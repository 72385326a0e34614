"""cdprobe_allreduce_ring without a GPU: the declared and exported symbol, its fault option, path constant and encoder,
the argument errors, the wrapper, the steps and faults of the Python restatement, the flags and ring-area layout of
probe_types.h against it, the compiled kernel's flag stores, polls and spills, and the Go mirror."""
import ctypes as C
import os
import re

import pytest

import allreduce_ring_ref as ref
import bwcurve_ref
from conftest import ROOT
from harness import FakeLib, c_tool, declared_symbols, exported_symbols, fake_probe, header_values
from kernel_tools import kernel_sass, ptxas_report

HEADER = os.path.join(ROOT, "include", "cdprobe.h")
U64_MAX = (1 << 64) - 1


def test_option_path_and_symbol_match_the_header(pkg, tmp_path):
    a = pkg.abi
    out = header_values(tmp_path, "CDPROBE_OPT_ALLREDUCE_RING_FAULT", "CDPROBE_ALLREDUCE_PATH_RING")
    assert out == [a.OPT_ALLREDUCE_RING_FAULT, a.ALLREDUCE_PATH_RING] == [23, 4]
    assert a.SYMBOLS["cdprobe_allreduce_ring"] == a.SYMBOLS["cdprobe_allreduce"]


def test_the_symbol_is_declared_and_exported_and_the_abi_set_still_matches(pkg):
    exported = exported_symbols(pkg.abi.LIB_PATH)
    declared = declared_symbols()
    assert "cdprobe_allreduce_ring" in declared and "cdprobe_allreduce_ring" in exported
    assert declared == set(pkg.abi.SYMBOLS)


def test_the_fault_encoder_and_its_refusals(pkg):
    a = pkg.abi
    assert a.allreduce_ring_fault(2, 5, 77) == (3 << 32) | (6 << 24) | 77
    assert a.allreduce_ring_fault(0, 0, 9, phase=1, mode=1) == (1 << 48) | (1 << 40) | (1 << 32) | (1 << 24) | 9
    assert a.allreduce_ring_fault(1, 2, 2000, mode=2) == (2 << 48) | (2 << 32) | (3 << 24) | 2000
    assert a.allreduce_ring_fault(15, 23, (1 << 24) - 1, 1, 2) >> 50 == 0
    for bad in (dict(mode=3), dict(mode=-1), dict(phase=2), dict(phase=-1), dict(arg=1 << 24), dict(arg=-1),
                dict(sender=255), dict(sender=-1), dict(k=255), dict(k=-1)):
        args = dict(sender=0, k=0, arg=0, phase=0, mode=0)
        args.update(bad)
        with pytest.raises(ValueError):
            a.allreduce_ring_fault(**args)


# ---- errors without a GPU -------------------------------------------------------------------------------------------
def test_a_null_handle_and_bad_reps_are_refused_and_fill_out(pkg):
    a = pkg.abi
    lib = a.load_library()
    t = a.AllReduceT()
    t.n, t.call_seq, t.n_sizes, t.measured[0], t.bad_words[0][0] = 77, 5, 3, 1, 9
    assert lib.cdprobe_allreduce_ring(None, 0, C.byref(t)) == a.ERR_ARG
    assert (t.abi, t.n, t.reps, t.call_seq, t.n_sizes, t.row_mask) == (2, 0, a.ALLREDUCE_DEFAULT_REPS, 0, 0, 0)
    assert sum(t.measured) == 0 and t.bad_words[0][0] == 0
    assert lib.cdprobe_allreduce_ring(None, 0, None) == a.ERR_ARG
    for reps in (1, a.ALLREDUCE_MAX_REPS + 1, 2 ** 32 - 1):
        t = a.AllReduceT()
        assert lib.cdprobe_allreduce_ring(None, reps, C.byref(t)) == a.ERR_ARG
        assert (t.abi, t.reps) == (2, reps) and sum(t.measured) == 0
    assert lib.cdprobe_set_option(None, a.OPT_ALLREDUCE_RING_FAULT, 1) == a.ERR_ARG


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
        def cdprobe_allreduce_ring(self, h, reps, out):
            calls.append((h.value, reps))
            t = out._obj
            t.abi, t.n, t.row_mask, t.reps, t.call_seq, t.n_sizes, t.path = 2, 3, 2, reps or 8, 4, 2, 4
            t.size[0], t.size[1] = 4096, 8192
            t.measured[1], t.measured[2] = 1, 1
            t.status[0], t.status[1], t.status[2] = a.ERR_STATE, a.ERR_INTEGRITY, a.ERR_TIMEOUT
            t.ns_min[1][0], t.ns_median[1][0], t.ns_max[1][0] = 1.0, 2.0, 3.0
            t.ns_median[1][1], t.sum[1][1], t.xr[1][1] = 4.0, 7, 9
            t.bad_words[1][1], t.first_bad[1][0], t.first_bad[1][1] = 1, U64_MAX, 8
            t.t0_ns[1], t.peak_gbps[1], t.half_bytes[1], t.bad_sizes[1] = 2.0, 2048.0, 4096, 2
            return a.ERR_ARG if reps > 64 else a.OK

    with fake_probe(pkg, Lib()) as p:
        ar = p.AllReduceRing()
        assert calls[-1] == (0x1234, 0)
        assert type(ar) is pkg.AllReduce
        assert (ar.n, ar.row_mask, ar.reps, ar.call_seq, ar.path, ar.sizes) == (3, 2, 8, 4, a.ALLREDUCE_PATH_RING,
                                                                                 [4096, 8192])
        assert ar.measured == [False, True, True]
        assert ar.status == [a.ERR_STATE, a.ERR_INTEGRITY, a.ERR_TIMEOUT]
        assert ar.ns_median[1] == [2.0, 4.0] and ar.ns_min[1] == [1.0, 0.0]
        assert ar.ns_median[0] is None and ar.sum[2] is None
        assert ar.sum[1] == [0, 7] and ar.xr[1] == [0, 9]
        assert ar.bad_words[1] == [0, 1] and ar.first_bad[1] == [U64_MAX, 8]
        p.AllReduceRing(reps=3)
        assert calls[-1] == (0x1234, 3)
        with pytest.raises(pkg.ProbeError) as e:
            p.AllReduceRing(65)
        assert e.value.code == a.ERR_ARG


# ---- the restatement ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", range(1, 17))
def test_the_steps_reduce_every_chunk_at_its_owner_and_deliver_it_everywhere(n):
    """A symbolic run of the steps: what each rank holds of each chunk is the set of inputs summed into it."""
    held = [[{g} for _ in range(n)] for g in range(n)]  # held[g][c]: the inputs rank g's copy of chunk c sums
    for s in range(n - 1):
        sent = [(g, ref.pushed_chunk(n, g, s, 0), set(held[g][ref.pushed_chunk(n, g, s, 0)])) for g in range(n)]
        for g, c, v in sent:
            assert c != g
            held[(g + 1) % n][c] = v | {(g + 1) % n}  # the receiver adds its own input at its next step
    for c in range(n):
        assert held[c][c] == set(range(n)), (n, c)
    full = [[held[g][c] if g == c else None for c in range(n)] for g in range(n)]
    for s in range(n - 1):
        sent = [(g, ref.pushed_chunk(n, g, s, 1), full[g][ref.pushed_chunk(n, g, s, 1)]) for g in range(n)]
        for g, c, v in sent:
            assert v == set(range(n)), (n, g, s, c)  # only a full chunk is ever pushed on
            full[(g + 1) % n][c] = v
    assert all(full[g][c] == set(range(n)) for g in range(n) for c in range(n))
    for g in range(n):
        assert ref.pushes(n, g, 0) == (set(range(n)) - {g} if n > 1 else set())
        assert ref.pushes(n, g, 1) == (set(range(n)) - {(g + 1) % n} if n > 1 else set())
        for c in ref.pushes(n, g, 0):
            assert ref.partial_ranks(n, g, c)[-1] == g and len(ref.partial_ranks(n, g, c)) == (g - 1 - c) % n + 1


@pytest.mark.parametrize("n", [2, 3, 5, 8, 16])
def test_failing_rows_run_from_the_hop_to_the_rank_before_the_owner(n):
    size = 64 * 8192
    for word in (0, 5 * 1024 + 3, size // 8 - 1):
        c = ref.chunk_of(size, n, word)
        for sender in range(n):
            assert ref.failing_rows(n, sender, 0, size, word) == list(range(n))
            if c == (sender + 1) % n:
                continue  # the sender does not push this chunk in the all-gather
            rows = ref.failing_rows(n, sender, 1, size, word)
            assert rows[0] == (sender + 1) % n and rows[-1] == (c - 1) % n and c not in rows
            assert len(rows) == len(set(rows))
            if sender == c:
                assert len(rows) == n - 1


# ---- flags and layout -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def helper(tmp_path_factory):
    return c_tool(tmp_path_factory, "ring_flags.cc")


def test_the_flag_grain_and_the_barrier_lines(helper):
    assert helper(["G"]) == [[1, 76 << 10]]


def test_flags_are_never_zero_and_distinct_within_a_call_and_from_the_call_before(helper):
    """Every (k < 24, r <= 64, phase) of one call and of the next, for call numbers across the 2^16 wrap."""
    calls = [1, 2, 255, 256, 65534, 65535, 65536, 65537, 131071, 131072, (1 << 40) + 65535]
    cases = [(c, k, r, ph) for c in calls for k in range(24) for r in range(65) for ph in (0, 1)]
    got = [v[0] for v in helper([f"F {c} {k} {r} {ph}" for c, k, r, ph in cases])]
    flags = {}
    for (c, k, r, ph), f in zip(cases, got):
        assert f == ref.flag(c, k, r, ph) and f != 0 and f < 1 << 32
        flags.setdefault(c, set()).add(f)
    for c in calls:
        assert len(flags[c]) == 24 * 65 * 2, c
        if c + 1 in flags:
            assert not flags[c] & flags[c + 1], c


def test_the_flag_offsets_tile_the_area_for_every_domain_and_ladder(helper):
    bpps = sorted({128, 4096 - 128, 4096, 4224, 16512, 24704, 57 * 8192 + 384, 1 << 20, 1 << 30, 32 << 30} |
                  {1 << e for e in range(7, 36)})
    lines, want = [], []
    for n in range(1, 17):
        for bpp in bpps:
            s_max = bwcurve_ref.ladder(bpp)[-1]
            U = ref.units(s_max)
            for u in sorted({0, 1, U // 2, U - 1}):
                lines.append(f"O {n} {s_max} {u}")
                want.append((s_max, U, u))
    for (s_max, U, u), (off, first, area) in zip(want, helper(lines)):
        assert (off, first, area) == (ref.flag_off(s_max, u), ref.flags_off(s_max), ref.area_bytes(s_max))
        assert s_max <= first < s_max + 128 and first % 128 == 0 and off % 4 == 0
        assert off == first + 4 * u and first + 4 * U == area  # one flag per unit, back to back, ending the area
    assert ref.area_bytes(32 << 30) == (32 << 30) + 4 * (4 << 20)


def test_bus_bandwidth_is_the_algorithm_bandwidth_times_2_n_minus_1_over_n():
    assert ref.busbw(100.0, 1) == 0.0 and ref.busbw(100.0, 2) == 100.0 and ref.busbw(100.0, 8) == 175.0


# ---- the compiled kernel ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kernel(pkg):
    return kernel_sass(pkg.abi.LIB_PATH, r"^_ZN3cdp21allreduce_ring_kernelE")[1]


def test_the_flag_store_is_a_system_scope_release_and_the_poll_a_strong_system_scope_load(kernel):
    """st.release.sys.global.u32 compiles to a MEMBAR.ALL.SYS and a 32-bit STG.E.STRONG.SYS, and ld.acquire.sys.global.u32
    to a 32-bit LDG.E.STRONG.SYS; the barrier lines' stores and polls are the 64-bit ones.  No TMA copy."""
    stores = [i for i, t in enumerate(kernel) if re.match(r"(@!?U?P\w+ )?STG\.E\.STRONG\.SYS ", t)]
    assert stores, "no 32-bit system-scope store"
    for i in stores:
        assert any(re.search(r"MEMBAR\.(ALL|SC)\.SYS", t) for t in kernel[max(0, i - 4):i]), kernel[i - 4:i + 1]
    assert any(re.match(r"(@!?U?P\w+ )?LDG\.E\.STRONG\.SYS ", t) for t in kernel)
    assert not any(t.startswith(("UBLKCP", "SYNCS.PHASECHK")) or " UBLKCP" in t for t in kernel)


def test_ptxas_reports_no_spills_in_the_ring_unit():
    props = ptxas_report("allreduce_ring_kernels.cu")
    ring = [k for k in props if "allreduce_ring_kernelE" in k]
    assert len(ring) == 1, props
    assert props[ring[0]][1:] == (0, 0), props



# ---- Go mirror ----------------------------------------------------------------------------------------------------
def test_go_ring_is_consistent_across_shim_stub_and_header():
    go = os.path.join(ROOT, "integration", "pkg", "fabricprobe")
    shim = open(os.path.join(go, "fabricprobe.go")).read()
    stub = open(os.path.join(go, "fabricprobe_stub.go")).read()
    assert "func (p *Probe) AllReduceRing(reps int) (AllReduce, error)" in shim
    assert "func (*Probe) AllReduceRing(int) (AllReduce, error)" in stub
    # optional binding: a missing symbol does not fail cdp_load, and AllReduceRing reports ErrUnsupported
    assert 'dlsym(cdp_dl, "cdprobe_allreduce_ring")' in shim and "cdp_has_allreduce_ring() == 0" in shim
    required = re.search(r"if \(!cdp_open[^)]*\)", shim).group(0)
    assert "cdp_arring" not in required
    # the ring converts its result through the same function, without adding to the strings other tests count
    assert "ring := allReduceOf(res)" in shim
    assert shim.count(" allReduceOf(ar)") == 3 and shim.count("return allReduceOf(ar), nil") == 2
    hdr = open(HEADER).read()
    assert "CDPROBE_API int cdprobe_allreduce_ring(cdprobe_t* h, uint32_t reps, cdprobe_allreduce_t* out);" in hdr
    assert re.search(r"#define CDPROBE_OPT_ALLREDUCE_RING_FAULT 23u", hdr)
    assert re.search(r"#define CDPROBE_ALLREDUCE_PATH_RING 4u", hdr)
