"""Domains of 9 to 16 ranks, and processes that drive several ranks each, against the oracle on the device.

The ABI allows CDPROBE_MAX_GPUS = 16 ranks and every device-side table is sized for 16, but the other GPU files stop
at 8 ranks and give each process one rank.  Code that only a wider domain reaches: the pingpong round field (N = 9 has
9 rounds), landing slot and source slice 15, per-issuer cell arrays filled to 16, the full diagnose candidate table
(writers 8 to 15), the longest phase table the schedule accepts, and, with several ranks per process, every index of
the form `rank * n_local + li` (first local rank, the fd exchange, the pingpong status merge).

- a. One process, N in {9, 12, 15, 16}, all on GPU 0 with 4 CTAs per rank (64 resident CTAs at N = 16): runs of every
  schedule against the oracle, the traced phase table against cdprobe_schedule, the stamps and the verdict; the phase
  table that overflows is refused at open and leaks nothing; every cell word for word; diagnose reports that name
  writers 8 to 15; landing faults on slots 14 and 15; the on-demand measurements; seeded model walks.
- b. Several processes, several ranks each (2 x 8, 2 x 4, 3 x 3), on GPU 0 with fd handles: the gathered matrix, the
  verdict, diagnose, the measurements' row masks and digests (every all-reduce's rows and the all-to-all's and memcpy's
  cells against their references in every process), a landing fault across processes, the pingpong status merge,
  and the refusals of mismatched and oversized domains.

More than 8 ranks in one process put more than 8 streams on one device; every such test runs in a child process whose
environment sets CUDA_DEVICE_MAX_CONNECTIONS=32 (include/cdprobe.h, CDPROBE_FLAG_ALLOW_SAME_DEVICE), since the test
process may have created its CUDA context already.  No test aborts a run or arms a short watchdog.
"""
import ctypes as C
import dataclasses
import json
import os
import random
import subprocess
import sys
import textwrap
import uuid

import pytest

import allreduce_ll_ref
import allreduce_ref
import alltoall_ref
import atomics_ref
import bwcurve_ref
import ce_alltoall_ref
import handle_model as hm
import test_ce_alltoall_gpu as ce_test
import latency_ref
import memcpy_ref
import pingpong_ref
import verdict_ref
import word_ref as ref
from conftest import ROOT
from test_bwcurve_gpu import assert_all_clean as assert_bwcurve_clean, slice_first_word
from test_gpu_parity import check_full_parity
from test_handle_sequences_gpu import Driver, walk
from test_latency_gpu import assert_clean as assert_latency_clean, first_word as latency_first_word
from test_latency_gpu import want_digest as latency_digest
from test_pingpong_gpu import assert_all_clean as assert_pingpong_clean, want as pingpong_want
from test_atomics_gpu import assert_all_clean as assert_atomics_clean
from test_timing_gpu import check_stamps, traces_of
from test_words_gpu import assert_report, observed, plant, region_offset, sweep, want_dict

pytestmark = pytest.mark.gpu

SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
LOCAL_DIAG = 0x04
SIMULATE_MIG = 0x200
UNI, SERIAL, ALL_RANK, PAIR = 0x80, 0x100, 0x400, 0x800
ERR_ARG, ERR_UNSUPPORTED, ERR_INTEGRITY = -2, -8, -10
G = ref.GRANULE_WORDS
CTAS = 4
# bytes_per_pair = NBYTES / (n - 1) rounded down to 128 B in sliced mode, NBYTES in full mode: not a whole number of
# 16 KiB granules at any n below, so the last granule of every region is partial (checked in wide_bpp)
NBYTES = (2 << 20) + 3 * 1024 + 384
WIDE = [9, 12, 15, 16]
SCHEDULES = {"default": 0, "unidirectional": UNI, "serial-verify": SERIAL, "local-diag": LOCAL_DIAG,
             "all-rank-barriers": ALL_RANK, "pair-barriers": PAIR}
# the longest phase table cdprobe_schedule accepts at N = 16; UNIDIRECTIONAL | SERIAL_VERIFY overflows from N = 13
LONGEST = UNI | LOCAL_DIAG
OVERFLOW = UNI | SERIAL
HOPS, LAT_REPS, ATOMIC_OPS, AT_REPS, BW_REPS = 64, 2, 64, 2, 2
# A pingpong digest xors every echo word of reps 0 .. reps: an odd count of them keeps the call and round fields in it
# (an even count cancels them), so a round field too narrow for 9 or more rounds changes the digest.
TRIPS, PP_REPS = 15, 2
MP_TRIPS = 9


def open_wide(pkg, n, flags=0, mode=1, nbytes=NBYTES):
    cfg = pkg.Config(ordinals=[0] * n, bytes=nbytes, mode=mode, flags=SAME | flags, ctas=CTAS, timeout_ms=20000)
    return cfg, pkg.Open(cfg)


def wide_bpp(pkg, n, flags=0, mode=1):
    bpp = pkg.plan(n, NBYTES, mode, flags).bytes_per_pair
    assert bpp % (G * 8), (n, mode, bpp)
    return bpp


# ---- the child process ----------------------------------------------------------------------------------------
CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path[:0] = [%r, %r]
    sys.modules["torch"] = None  # not needed here; conftest.gpu_count() then reports 0, which only feeds skip marks
    import cdprobe_pkg
    from oracle import oracle
    import test_wide_domains_gpu as t
    pkg = cdprobe_pkg.load()
    getattr(t, sys.argv[1])(pkg, oracle, *json.loads(sys.argv[2]))
    print("CHILD OK")
    """
) % (ROOT, os.path.join(ROOT, "tests"))


def in_child(case, *args, timeout=1200):
    """Run case(pkg, oracle, *args) in a fresh process with 32 hardware queues per device; its assertion is the
    failure message."""
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    pr = subprocess.run([sys.executable, "-c", CHILD, case, json.dumps(args)], env=env, capture_output=True, text=True,
                        timeout=timeout)
    assert pr.returncode == 0 and "CHILD OK" in pr.stdout, pr.stderr[-8000:]


# ---- checks of one run -----------------------------------------------------------------------------------------
def schedule_flags(cfg_flags):
    """The flags cdprobe_schedule is asked for: the overlapped verify is on unless the serial one is."""
    return cfg_flags if cfg_flags & SERIAL else cfg_flags | hm.FLAG_OVERLAP_VERIFY


def check_phases(pkg, p, traces, n, flags, mode):
    """Every local rank's traced phases are cdprobe_schedule's table for it (kinds, peers and barrier masks), and its
    read peers come in the order of cdprobe_plan's partner table."""
    sched = hm.schedule_fn(p._lib, pkg.abi)
    info = p.Info()
    pl = pkg.plan(n, NBYTES, mode, flags)
    for li in range(info.n_local):
        g = info.first_local_rank + li
        tr = traces[g]
        s = sched(n, g, NBYTES, mode, 3, schedule_flags(flags), info.ctas[li], 32)
        assert len(tr) == s.n_phases <= pkg.abi.MAX_PHASES, (g, len(tr), s.n_phases)
        for k, ph in enumerate(tr):
            want = {"job0": hm.KIND_NAMES[s.kind[0][k]], "peer0": s.peer[0][k], "job1": hm.KIND_NAMES[s.kind[1][k]],
                    "peer1": s.peer[1][k], "sync_all": s.sync_all[k], "sync_mask": s.sync_mask[k],
                    "post_mask": s.post_mask[k]}
            assert {f: ph[f] for f in want} == want, (g, k, ph, want)
        reads = [ph["peer0"] for ph in tr if ph["job0"] == "read" and ph["peer0"] != g]
        partners = [pl.partner[r][g] for r in range(pl.rounds) if pl.partner[r][g] >= 0]
        assert reads == partners, (g, reads, partners)


def check_run(pkg, oracle, p, cfg, res, n, flags, mode):
    diag = bool(flags & LOCAL_DIAG)
    assert res.n == n and res.row_mask == (1 << n) - 1 and not res.aborted
    assert res.reach == [[1] * n for _ in range(n)]
    check_full_parity(pkg, oracle, res, n, NBYTES, mode, 3, diag)
    traces = traces_of(p)
    check_phases(pkg, p, traces, n, flags, mode)
    check_stamps(res, traces)
    verdict_ref.check(res, traces, 3, diag, pkg.gate(cfg, n))
    return traces


# ---- a1 / a3. runs of every schedule, and every cell word for word -------------------------------------------------
def case_runs(pkg, oracle, n):
    for name, flags in SCHEDULES.items():
        cfg, p = open_wide(pkg, n, flags)
        with p:
            for run in (1, 2):
                r = p.Run()
                check_run(pkg, oracle, p, cfg, r, n, flags, 1)
            if name in ("default", "local-diag"):
                sweep(p, oracle, r, NBYTES, 1, f"n {n}, {name}", diag=bool(flags & LOCAL_DIAG))
    cfg, p = open_wide(pkg, n, mode=2)
    with p:
        for run in (1, 2):
            check_run(pkg, oracle, p, cfg, p.Run(), n, 0, 2)
        sweep(p, oracle, p.Run(), NBYTES, 2, f"n {n}, full")


def longest_accepted_table(pkg, n):
    """The most phases any rank's table has under any schedule flags cdprobe_schedule accepts at n ranks."""
    sched, s, most = pkg.abi.load_library().cdprobe_schedule, pkg.abi.ScheduleT(), 0
    for bits in range(32):
        flags = sum(f for k, f in enumerate((UNI, SERIAL, ALL_RANK, PAIR, LOCAL_DIAG)) if bits >> k & 1)
        for g in range(n):
            if sched(n, g, NBYTES, 1, 3, schedule_flags(flags), CTAS, 32, C.byref(s)) == 0:
                most = max(most, s.n_phases)
    return most


def case_paths_and_longest_table(pkg, oracle):
    n = 16
    for flags in (0, LOCAL_DIAG):
        cfg, p = open_wide(pkg, n, flags)
        with p:
            for path in (0, 1, 2):
                p.SetOption(pkg.abi.OPT_PATH, path)
                for run in (1, 2):
                    r = p.Run()
                    check_run(pkg, oracle, p, cfg, r, n, flags, 1)
                sweep(p, oracle, r, NBYTES, 1, f"n 16, flags {flags:#x}, path {path}", diag=bool(flags & LOCAL_DIAG))
    cfg, p = open_wide(pkg, n, LONGEST)
    with p:
        for path in (0, 1, 2):
            p.SetOption(pkg.abi.OPT_PATH, path)
            for run in (1, 2):
                r = p.Run()
                check_run(pkg, oracle, p, cfg, r, n, LONGEST, 1)
            assert r.phases == longest_accepted_table(pkg, n), r.phases
        sweep(p, oracle, r, NBYTES, 1, "n 16, longest table", diag=True)


@pytest.mark.parametrize("n", WIDE)
def test_runs_of_every_schedule_equal_the_oracle(pkg, oracle, n):
    for mode in (1, 2):
        wide_bpp(pkg, n, mode=mode)
    in_child("case_runs", n)


def test_sixteen_ranks_every_path_and_the_longest_table(pkg, oracle):
    in_child("case_paths_and_longest_table")


# ---- a2. the table that overflows is refused at open ---------------------------------------------------------------
_primary = {}


def device_free_bytes():
    """Free memory of GPU 0 from the driver (cuMemGetInfo in its primary context, which this process keeps)."""
    cu = C.CDLL("libcuda.so.1")
    if not _primary:
        dev, ctx = C.c_int(), C.c_void_p()
        assert cu.cuInit(0) == 0 and cu.cuDeviceGet(C.byref(dev), 0) == 0
        assert cu.cuDevicePrimaryCtxRetain(C.byref(ctx), dev) == 0
        _primary["ctx"] = ctx
    assert cu.cuCtxPushCurrent_v2(_primary["ctx"]) == 0
    free, total = C.c_size_t(), C.c_size_t()
    assert cu.cuMemGetInfo_v2(C.byref(free), C.byref(total)) == 0
    assert cu.cuCtxPopCurrent_v2(C.byref(C.c_void_p())) == 0
    return free.value


# Large enough that a refused open which kept its allocations would show: 16 ranks x (24 MiB of source + 24 MiB of
# landing slots + 2 MiB of control) = 800 MiB per open, under 1 GiB.
REFUSED_BYTES = 24 << 20
REFUSALS = 3
LEAK_TOLERANCE = 512 << 20  # other contexts on the device may allocate meanwhile; a leak would be 2.4 GB


def case_overflow_refused(pkg, oracle, n):
    with pkg.Open(pkg.Config(ordinals=[0], bytes=1 << 20)) as p:  # the context exists before the first reading
        p.Run()
    before = device_free_bytes()
    cfg = pkg.Config(ordinals=[0] * n, bytes=REFUSED_BYTES, flags=SAME | OVERFLOW, ctas=CTAS, timeout_ms=20000)
    for _ in range(REFUSALS):
        with pytest.raises(pkg.ProbeError) as e:
            pkg.Open(cfg)
        assert e.value.code == ERR_ARG, (e.value.code, str(e.value))
    after = device_free_bytes()
    assert before - after < LEAK_TOLERANCE, (before, after)
    # the same process opens the same domain with the overlapped verify, and it runs at parity
    cfg.flags = SAME | UNI
    with pkg.Open(cfg) as p:
        r = p.Run()
        assert r.reach == [[1] * n for _ in range(n)] and not r.aborted
        check_full_parity(pkg, oracle, r, n, REFUSED_BYTES, 1, 3)


@pytest.mark.parametrize("n", [13, 16])
def test_overflowing_table_is_refused_at_open_and_leaks_nothing(pkg, oracle, n):
    rc = pkg.abi.load_library().cdprobe_schedule(n, 0, REFUSED_BYTES, 1, 3, OVERFLOW, CTAS, 32,
                                                  C.byref(pkg.abi.ScheduleT()))
    assert rc == ERR_ARG  # the table itself (test_schedule.py); here: cdprobe_open passes the refusal on
    in_child("case_overflow_refused", n)


# ---- a4. diagnose at full width --------------------------------------------------------------------------------
def case_diagnose_full_width(pkg, oracle):
    n, flags = 16, LOCAL_DIAG
    rng = random.Random(16)
    cfg, p = open_wide(pkg, n, flags)
    with p:
        r = p.Run()
        W = r.bytes_per_pair // 8
        i, j = 0, 15
        off = region_offset(oracle, n, NBYTES, 1, True, "write", i, j)
        spots = sorted(rng.sample(range(1, W // G * G), 20)) + [W // G * G + 7, W - 1]  # the partial granule too
        # three runs, each arming at most 8 words (kMaxLandingFaults): every other writer into rank 15 (1 .. 15, the
        # loop-back writer included), then a STALE, a DISPLACED and a FLIP word
        plans = [[("foreign", w) for w in range(1, 8)], [("foreign", w) for w in range(8, 16)],
                 [("stale", 3), ("displaced", None), ("flip", None), ("foreign", 9), ("foreign", 14)]]
        used = 0
        for batch in plans:
            seq = r.run_seq + 1  # the run that writes the slot next
            spec = ref.write_spec(SEED, n, i, j, seq, W)
            exp = spec.expected()
            faults = []
            for kind, arg in batch:
                k = spots[used]
                used += 1
                if kind == "foreign":
                    word = int(ref.write_words(ref.write_salt(SEED, arg, j, seq), rng.randrange(W), 1)[0])
                elif kind == "stale":
                    word = int(ref.write_words(ref.write_salt(SEED, i, j, seq - arg), rng.randrange(W), 1)[0])
                elif kind == "displaced":
                    word = int(exp[(k + 1 + rng.randrange(W - 1)) % W])
                else:
                    word = int(exp[k]) ^ (1 << rng.randrange(64))
                faults.append((k, int(exp[k]) ^ word))
            p.CorruptLanding(i, j, faults)
            r = p.Run()
            assert r.run_seq == seq and r.reach_write[i][j] == 0 and not r.aborted
            want = want_dict(spec, observed(spec, faults), "write", i, seq, off)
            kinds = want["kind_count"]
            if batch[0][0] == "foreign":
                assert kinds[ref.FOREIGN] == len(batch), kinds
            else:
                assert kinds[ref.STALE] == kinds[ref.DISPLACED] == kinds[ref.FLIP] == 1 and kinds[ref.FOREIGN] == 2
            for reader in (j, i):
                assert_report(p.Diagnose("write", i, j, reader=reader), want, (batch, reader))
        p.CorruptLanding(i, j, [])
        # a read slice of rank 0 that holds words of ranks 9 .. 15: the slice rank 15 reads
        r = p.Run()
        assert r.reach == [[1] * n for _ in range(n)]
        first = oracle.lib().cdoracle_slot(15, 0) * W
        pl = pkg.plan(n, NBYTES, 1, flags)
        spec = ref.read_spec(SEED, n, 0, first, W, pl.src_bytes // 8)
        idx = sorted(rng.sample(range(W), 21))
        faults = plant(p, 0, 8 * first, spec, rng, idx, ["foreign", "foreign", "foreign", "zero", "flip", "displaced"],
                       tuple(range(9, 16)))
        want = want_dict(spec, observed(spec, faults), "read", 15, r.run_seq,
                         region_offset(oracle, n, NBYTES, 1, True, "read", 15, 0))
        assert want["kind_count"][ref.FOREIGN] >= 10
        assert {s["rank"] for s in want["sample"] if s["kind"] == ref.FOREIGN} <= set(range(9, 16))
        for reader in (15, 0):
            assert_report(p.Diagnose("read", 15, 0, reader=reader), want, reader)
        for k, mask in faults:
            p.Corrupt(0, 8 * (first + k), mask)
        r = p.Run()
        check_run(pkg, oracle, p, cfg, r, n, flags, 1)


def test_diagnose_names_writers_and_owners_past_rank_8(pkg, oracle):
    in_child("case_diagnose_full_width")


# ---- a5. landing faults on the last slots ------------------------------------------------------------------------
def case_landing_faults(pkg, oracle):
    n, flags = 16, LOCAL_DIAG
    cfg, p = open_wide(pkg, n, flags)
    with p:
        W = p.Info().bytes_per_pair // 8
        faults = [(0, 1 << 63), (W - 1, 0xF0), (W // G * G + 5, 1 << 7)]
        for path in (0, 1, 2):
            p.SetOption(pkg.abi.OPT_PATH, path)
            for i, j in ((15, 14), (14, 15), (15, 15)):
                p.CorruptLanding(i, j, faults)
                r = p.Run()
                want_w = [[0 if (a, b) == (i, j) else 1 for b in range(n)] for a in range(n)]
                assert r.reach_write == want_w and r.reach_read == [[1] * n for _ in range(n)], (path, i, j)
                assert not r.aborted
                for a in range(n):
                    for b in range(n):  # the writer's checksum is the oracle's, the armed cell's too
                        assert (r.sum_write[a][b], r.xor_write[a][b]) == \
                            oracle.write_checksum(SEED, a, b, r.run_seq, W), (path, i, j, a, b)
                traces = traces_of(p)
                check_stamps(r, traces)
                verdict_ref.check(r, traces, 3, True, pkg.gate(cfg, n))
                p.CorruptLanding(i, j, [])
                check_run(pkg, oracle, p, cfg, p.Run(), n, flags, 1)


def test_landing_faults_on_slots_14_and_15_fail_exactly_their_cell(pkg, oracle):
    in_child("case_landing_faults")


# ---- a6. the on-demand measurements --------------------------------------------------------------------------------
def case_measurements(pkg, oracle, n, flags):
    diag = bool(flags & LOCAL_DIAG)
    cfg, p = open_wide(pkg, n, flags)
    with p:
        bpp = p.Info().bytes_per_pair
        lat = p.Latency(hops=HOPS, reps=LAT_REPS)
        assert lat.row_mask == (1 << n) - 1
        for i in range(n):
            for j in range(n):
                if i == j and not diag:
                    assert not lat.measured[i][j]
                    continue
                assert_latency_clean(lat, i, j)
                assert lat.digest[i][j] == latency_digest(oracle, lat, n, 1, i, j), (i, j)

        pp = p.PingPong(trips=TRIPS, reps=PP_REPS)
        assert (pp.row_mask, pp.call_seq) == ((1 << n) - 1, 1)
        assert_pingpong_clean(pkg, pp)
        if n == 16:
            ini, tgt, trip = 15, 14, 5  # initiator 16, target 15 in the option's 1-based encoding
            p.SetOption(pkg.abi.OPT_PINGPONG_FAULT, (16 << 32) | (15 << 16) | trip)
            pp = p.PingPong(trips=TRIPS, reps=PP_REPS)
            assert pp.status[ini][tgt] == ERR_INTEGRITY
            assert pp.digest[ini][tgt] == pingpong_want(pkg, pp, ini, tgt, fault_trip=trip) != pingpong_want(pkg, pp, ini, tgt)
            assert_pingpong_clean(pkg, pp, skip={(ini, tgt)})
            p.SetOption(pkg.abi.OPT_PINGPONG_FAULT, 0)
            assert_pingpong_clean(pkg, p.PingPong(trips=TRIPS, reps=PP_REPS))

        for kind in (atomics_ref.FETCH_ADD, atomics_ref.CAS, atomics_ref.CONTENDED):
            at = p.Atomics(kind, ops=ATOMIC_OPS, reps=AT_REPS)
            assert at.row_mask == (1 << n) - 1
            assert_atomics_clean(at, diag)
            if n == 16:
                for value, (i, j) in (((16 << 16) | 16, (15, 15)), ((16 << 16) | 1, (15, 0))):
                    p.SetOption(pkg.abi.OPT_ATOMICS_FAULT, value)
                    at = p.Atomics(kind, ops=ATOMIC_OPS, reps=AT_REPS)
                    assert at.status[i][j] == ERR_INTEGRITY, (kind, i, j, at.status[i][j])
                    if kind != atomics_ref.CONTENDED:
                        assert at.digest[i][j] == atomics_ref.cell_digest(at.call_seq, kind, ATOMIC_OPS, AT_REPS, fault=True)
                    assert_atomics_clean(at, diag, skip={(i, j)})
                    p.SetOption(pkg.abi.OPT_ATOMICS_FAULT, 0)
                assert_atomics_clean(p.Atomics(kind, ops=ATOMIC_OPS, reps=AT_REPS), diag)

        bw = p.BwCurve(reps=BW_REPS)
        assert bw.row_mask == (1 << n) - 1
        assert_bwcurve_clean(bw, oracle, bpp, diag)
        if n == 16:
            sizes = bwcurve_ref.ladder(bpp)
            i, j = 14, 15
            base = slice_first_word(n, i, j, bpp, False) * 8
            for o in (40, bpp // 16384 * 16384 + 1000):
                p.Corrupt(j, base + o, 1 << 17)
                bw = p.BwCurve(reps=BW_REPS)
                assert bw.status[i][j] == ERR_INTEGRITY, o
                assert bw.bad_sizes[i][j] == sum(1 << k for k, s in enumerate(sizes) if s > o), (o, bw.bad_sizes[i][j])
                assert_bwcurve_clean(bw, oracle, bpp, diag, skip={(i, j)})
                p.Corrupt(j, base + o, 1 << 17)
            assert_bwcurve_clean(p.BwCurve(reps=BW_REPS), oracle, bpp, diag)
        # the copy-engine all-to-all: n ranks on one device need n x n streams (n x (n + 1) with the loop-back),
        # 81, 225 and 272 of the 32 this process has: refused with the need named, advancing nothing, and memcpy
        # then runs clean on the handle
        need, ordinal = ce_alltoall_ref.queues(n, diag, [0] * n)
        assert (n, need, ordinal) in ((9, 81, 0), (15, 225, 0), (16, 272, 0))
        for op in (pkg.abi.OP_READ, pkg.abi.OP_WRITE):
            rc, t = p.ce_alltoall_raw(op, 2)
            assert rc == ERR_UNSUPPORTED and t.call_seq == 0 and sum(t.measured) == 0, rc
            assert p._lib.cdprobe_last_error().decode() == \
                "cdprobe_ce_alltoall: " + ce_alltoall_ref.queue_message(need, 0, 32)
        mc = p.Memcpy(pkg.abi.OP_WRITE, reps=1)
        assert mc.call_seq == 1 and mc.sizes == bwcurve_ref.ladder(bpp)
        for g, j in ce_alltoall_ref.cells(n, diag):
            cell = memcpy_ref.cell(n, bpp, 1, pkg.abi.OP_WRITE, g, j)
            assert mc.measured[g][j] and mc.status[g][j] == 0 and mc.bad_sizes[g][j] == 0, (g, j)
            assert list(zip(mc.sum[g][j], mc.xr[g][j])) == \
                [tuple(e) for e in memcpy_ref.expected(oracle, SEED, cell, mc.sizes)], (g, j)
        r = p.Run()  # the measurements disturbed nothing
        check_run(pkg, oracle, p, cfg, r, n, flags, 1)


@pytest.mark.parametrize("n,flags", [(9, 0), (15, 0), (16, LOCAL_DIAG)], ids=["n9", "n15", "n16-local-diag"])
def test_measurements_of_every_cell(pkg, oracle, n, flags):
    in_child("case_measurements", n, flags)


# ---- a7. model walks ---------------------------------------------------------------------------------------------
WALK_STEPS = 40


def case_walk(pkg, oracle, n, seed):
    nbytes = (1 << 20) + 5 * 1024 + 128
    cfg = pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=CTAS, timeout_ms=20000)
    with pkg.Open(cfg) as p:
        walk(Driver(pkg, oracle, p, cfg, n, nbytes), seed, WALK_STEPS, ctas_cap=CTAS)


@pytest.mark.parametrize("n,seed", [(9, 91), (16, 161)])
def test_seeded_walk(pkg, oracle, n, seed):
    in_child("case_walk", n, seed)


# ---- b. several processes, several ranks each -------------------------------------------------------------------
MP_CHILD = textwrap.dedent(
    """
    import dataclasses, json, sys
    sys.path[:0] = [%r, %r]
    sys.modules["torch"] = None
    import cdprobe_pkg
    import test_wide_domains_gpu as t
    pkg = cdprobe_pkg.load()
    session, rank, world, n_local, what = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), sys.argv[5]
    print("RESULT " + json.dumps(t.mp_process(pkg, session, rank, world, n_local, what)))
    """
) % (ROOT, os.path.join(ROOT, "tests"))

MP_TIMEOUT_MS = 60000


def fields(obj):
    return {k: v for k, v in dataclasses.asdict(obj).items() if k != "raw"}


def mp_process(pkg, session, rank, world, n_local, what):
    """One process of a multi-process domain; returns what the parent checks."""
    flags = SAME | (SIMULATE_MIG if what == "mig" and rank == 1 else 0)
    if what == "mismatch":
        n_local += rank
    cfg = pkg.Config(ordinals=[0] * n_local, bytes=NBYTES, world_size=world, rank=rank, session=session, flags=flags,
                     ctas=CTAS, timeout_ms=MP_TIMEOUT_MS, link_peak_gbps=1e-3)
    if what in ("mismatch", "oversized"):
        try:
            pkg.Open(cfg).Close()
            return {"rc": 0}
        except pkg.ProbeError as e:
            return {"rc": e.code}
    out = {}
    with pkg.Open(cfg) as p:
        info = p.Info()
        out["info"] = {"first": info.first_local_rank, "n_local": info.n_local, "n": info.n,
                       "handle_type": info.handle_type}
        if what == "mig":  # one process's ranks are MIG instances: no pair with them is exchanged, in any process
            out["pp"] = fields(p.PingPong(trips=MP_TRIPS, reps=PP_REPS))
            return out
        n = info.n
        out["gate"] = pkg.gate(cfg, n)
        out["runs"] = []
        for _ in range(2):
            raw = pkg.abi.ResultT()
            assert p.run_raw(raw) == pkg.abi.OK
            pre = fields(pkg.Result.from_c(pkg.abi.ResultT.from_buffer_copy(raw)))
            assert p._lib.cdprobe_gather(p._h, C.byref(raw)) == pkg.abi.OK
            out["runs"].append({"pre": pre, "post": fields(pkg.Result.from_c(raw)),
                                "traces": {str(g): tr for g, tr in traces_of(p).items()}})
        local = range(info.first_local_rank, info.first_local_rank + info.n_local)
        out["diags"] = []
        for op in ("read", "write"):
            for i in range(n):
                for j in range(n):
                    for reader in (sorted({i, j} & set(local)) if i != j else []):
                        d = p.Diagnose(op, i, j, reader=reader)
                        out["diags"].append([op, i, j, reader, d.bad_words, d.bytes, d.run_seq, d.region_offset])
        out["lat"] = fields(p.Latency(hops=HOPS, reps=LAT_REPS))
        out["at"] = [fields(p.Atomics(k, ops=ATOMIC_OPS, reps=AT_REPS)) for k in range(3)]
        out["pp"] = fields(p.PingPong(trips=MP_TRIPS, reps=PP_REPS))
        out["bw"] = fields(p.BwCurve(reps=BW_REPS))
        out["ar"] = fields(p.AllReduce(reps=2))
        out["a2a"] = fields(p.AllToAll(reps=2))
        for key, fn in (("ts", p.AllReduceTwoShot), ("ll", p.AllReduceLL), ("ring", p.AllReduceRing),
                        ("push", p.AllReducePush)):
            out[key] = fields(fn(reps=2))
        out["mc"] = [fields(p.Memcpy(op, reps=2)) for op in (pkg.abi.OP_READ, pkg.abi.OP_WRITE)]
        out["ce"] = []
        for op in (pkg.abi.OP_READ, pkg.abi.OP_WRITE):
            rc, t = p.ce_alltoall_raw(op, 2)
            out["ce"].append({"rc": rc, "error": p._lib.cdprobe_last_error().decode() if rc else "",
                              **({} if rc else ce_test.as_dict(pkg.CeAllToAll.from_c(t)))})
        # a landing fault armed in process 0 on a cell whose target lives in the last process
        W = info.bytes_per_pair // 8
        if rank == 0:
            p.CorruptLanding(0, n - 1, [(0, 1), (W - 1, 1 << 40)])
        out["faulted"] = fields(p.Run(gather=True))
        if rank == 0:
            p.CorruptLanding(0, n - 1, [])
        out["healed"] = fields(p.Run(gather=True))
        try:
            p.UnmapPeer(0, (info.first_local_rank + info.n_local) % n)
            out["unmap"] = 0
        except pkg.ProbeError as e:
            out["unmap"] = e.code
        out["after_unmap"] = fields(p.PingPong(trips=MP_TRIPS, reps=PP_REPS))
    return out


def run_processes(world, n_local, what, timeout=900):
    """The processes of the "full" case have 32 hardware queues per device, so the copy-engine all-to-all runs up to 32
    streams on one; the others keep the runtime's default."""
    session = f"wd-{uuid.uuid4().hex[:12]}"
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32") if what == "full" else None
    procs = [subprocess.Popen([sys.executable, "-c", MP_CHILD, session, str(r), str(world), str(n_local), what],
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=env)
             for r in range(world)]
    outs = []
    for pr in procs:
        so, se = pr.communicate(timeout=timeout)
        assert pr.returncode == 0, se[-4000:]
        outs.append(json.loads([l for l in so.splitlines() if l.startswith("RESULT ")][-1][7:]))
    return outs


class AsResult:
    """A Result rebuilt from a child's JSON: the attributes the checks read."""

    def __init__(self, d):
        self.__dict__.update(d)
        self.reach = [[a & b for a, b in zip(ra, rb)] for ra, rb in zip(d["reach_read"], d["reach_write"])]


MP_SHAPES = [(2, 8), (2, 4), (3, 3)]


@pytest.mark.parametrize("world,n_local", MP_SHAPES, ids=[f"{w}x{k}" for w, k in MP_SHAPES])
def test_processes_with_several_ranks_each(pkg, oracle, world, n_local):
    n = world * n_local
    outs = run_processes(world, n_local, "full")
    W = wide_bpp(pkg, n) // 8
    pl = pkg.plan(n, NBYTES, 1)
    for rank, o in enumerate(outs):
        mine = set(range(rank * n_local, (rank + 1) * n_local))
        rows = sum(1 << g for g in mine)
        assert o["info"] == {"first": rank * n_local, "n_local": n_local, "n": n, "handle_type": 1}, o["info"]
        for k, run in enumerate(o["runs"]):
            assert run["pre"]["row_mask"] == rows
            post = AsResult(run["post"])
            assert post.row_mask == (1 << n) - 1 and post.reach == [[1] * n for _ in range(n)] and not post.aborted
            check_full_parity(pkg, oracle, post, n, NBYTES, 1, 3)
            traces = {int(g): tr for q in outs for g, tr in q["runs"][k]["traces"].items()}
            verdict_ref.check(post, traces, 3, False, tuple(o["gate"]))
            for g in mine:
                assert [ph["job0"] for ph in traces[g]] == [ph["job0"] for ph in run["traces"][str(g)]]
        assert o["runs"][1]["post"]["run_seq"] == o["runs"][0]["post"]["run_seq"] + 1
        # every cell a local rank can read diagnoses clean
        assert len(o["diags"]) == 2 * sum(len({i, j} & mine) for i in range(n) for j in range(n) if i != j)
        for op, i, j, reader, bad, nb, seq, off in o["diags"]:
            assert bad == 0 and nb == W * 8 and seq == o["runs"][1]["post"]["run_seq"], (rank, op, i, j, reader)
            assert off == region_offset(oracle, n, NBYTES, 1, False, op, i, j), (op, i, j)
        # the one-sided measurements fill exactly the local rows
        lat = o["lat"]
        assert lat["row_mask"] == rows
        for i in range(n):
            for j in range(n):
                assert lat["measured"][i][j] == (i in mine and i != j), (i, j)
                if lat["measured"][i][j]:
                    first = latency_first_word(oracle, n, 1, i, j, W * 8)
                    assert lat["status"][i][j] == 0
                    assert lat["digest"][i][j] == latency_ref.digest(SEED, i, j, first, W * 8 // latency_ref.LINE_BYTES,
                                                                     HOPS, LAT_REPS), (i, j)
        for k, at in enumerate(o["at"]):
            assert at["row_mask"] == rows and at["call_seq"] == k + 1
            for i in range(n):
                for j in range(n):
                    assert at["measured"][i][j] == (i in mine and i != j), (k, i, j)
                    if at["measured"][i][j]:
                        assert at["status"][i][j] == 0
                        assert at["digest"][i][j] == atomics_ref.cell_digest(at["call_seq"], k, ATOMIC_OPS, AT_REPS)
        # the collective measurements agree on call_seq in every process, and their cells are clean
        for key in ("pp", "bw"):
            assert o[key]["call_seq"] == outs[0][key]["call_seq"] == 1, key
        pp, bw = o["pp"], o["bw"]
        assert pp["row_mask"] == rows and bw["row_mask"] == rows
        assert bw["sizes"] == bwcurve_ref.ladder(W * 8)
        for i in range(n):
            for j in range(n):
                assert pp["measured"][i][j] == bw["measured"][i][j] == (i in mine and i != j), (i, j)
                if not pp["measured"][i][j]:
                    continue
                assert pp["status"][i][j] == 0 and bw["status"][i][j] == 0 and bw["bad_sizes"][i][j] == 0
                assert pp["digest"][i][j] == \
                    pingpong_ref.cell_digest(1, pl.partner, pl.rounds, i, j, MP_TRIPS, PP_REPS), (i, j)
                first = slice_first_word(n, i, j, W * 8, False)
                assert [[s, x] for s, x in zip(bw["sum"][i][j], bw["xr"][i][j])] == \
                    [list(oracle.src_checksum(SEED, j, first, s // 8)) for s in bw["sizes"]], (i, j)
        # the all-reduce fills exactly the local rows, and the all-to-all exactly the cells a local rank receives, with
        # the pattern's (S, X) at every size; both agree on call_seq in every process
        ar, a2a = o["ar"], o["a2a"]
        sizes = bwcurve_ref.ladder(W * 8)
        for key in ("ar", "a2a"):
            assert o[key]["call_seq"] == outs[0][key]["call_seq"] == 1 and o[key]["sizes"] == sizes, key
            assert o[key]["row_mask"] == rows and o[key]["reps"] == 2, key
        ar_want = [list(sx) for sx in allreduce_ref.expected(SEED, n, tuple(sizes))]
        for r in range(n):
            assert ar["measured"][r] == a2a["measured"][r] == (r in mine), r
            if r in mine:
                assert ar["status"][r] == 0 and ar["bad_sizes"][r] == 0 and ar["bad_words"][r] == [0] * len(sizes)
                assert [[s, x] for s, x in zip(ar["sum"][r], ar["xr"][r])] == ar_want, r
                assert a2a["status"][r] == 0 and a2a["blocks"][r] == n - 1, r
        for s in range(n):
            for d in range(n):
                assert a2a["cell_measured"][s][d] == (d in mine and s != d), (s, d)
                if a2a["cell_measured"][s][d]:
                    assert a2a["cell_status"][s][d] == 0 and a2a["bad_words"][s][d] == [0] * len(sizes), (s, d)
                    assert [[x, y] for x, y in zip(a2a["sum"][s][d], a2a["xr"][s][d])] == \
                        [list(e) for e in alltoall_ref.expected(SEED, s, d, 1, 2, sizes)], (s, d)
        # the two-shot, LL, ring and push fill exactly the local rows with the pattern's sums, on their own ladders and
        # paths; memcpy fills exactly the cells a local rank issues, with its source slice's (S, X), for both ops
        for key, ladder, path in (("ts", sizes, 0), ("ll", allreduce_ll_ref.ladder(W * 8), 3), ("ring", sizes, 4),
                                  ("push", sizes, 0)):
            got = o[key]
            assert got["call_seq"] == outs[0][key]["call_seq"] == 1 and got["sizes"] == ladder, key
            assert (got["row_mask"], got["reps"], got["path"]) == (rows, 2, path), key
            want = [list(sx) for sx in allreduce_ref.expected(SEED, n, tuple(ladder))]
            for r in range(n):
                assert got["measured"][r] == (r in mine), (key, r)
                if r in mine:
                    assert got["status"][r] == 0 and got["bad_sizes"][r] == 0, (key, r)
                    assert got["bad_words"][r] == [0] * len(ladder), (key, r)
                    assert [[s, x] for s, x in zip(got["sum"][r], got["xr"][r])] == want, (key, r)
        for call, mc in enumerate(o["mc"], 1):
            assert (mc["call_seq"], mc["row_mask"], mc["reps"], mc["sizes"]) == (call, rows, 2, sizes), mc["op"]
            for g in range(n):
                for d in range(n):
                    assert mc["measured"][g][d] == (g in mine and g != d), (mc["op"], g, d)
                    if mc["measured"][g][d]:
                        cell = memcpy_ref.cell(n, W * 8, 1, mc["op"], g, d)
                        assert mc["status"][g][d] == 0 and mc["bad_words"][g][d] == [0] * len(sizes), (g, d)
                        assert [[s, x] for s, x in zip(mc["sum"][g][d], mc["xr"][g][d])] == \
                            [list(e) for e in memcpy_ref.expected(oracle, SEED, cell, sizes)], (mc["op"], g, d)
        # the copy-engine all-to-all: n_local x n streams per process on one device.  2 x 8 needs 128 of 32 and is
        # refused in both processes, each naming its own need; 2 x 4 runs at exactly 32 and 3 x 3 at 27, every block
        # checked by its owner's process and clean
        need, _ = ce_alltoall_ref.queues(n, False, [0] * n_local)
        assert need == n_local * n
        for call, ce in enumerate(o["ce"], 1):
            if need > 32:
                assert ce == {"rc": ERR_UNSUPPORTED, "error": "cdprobe_ce_alltoall: " +
                              ce_alltoall_ref.queue_message(need, 0, 32)}, ce
                continue
            assert ce["rc"] == 0 and ce["call_seq"] == call and ce["row_mask"] == rows, ce["rc"]
            ce_test.check_call(ce, oracle, W * 8, 1, False)
            for g, j in ce_alltoall_ref.cells(n, False):
                assert ce["cell_measured"][g][j] == (ce_alltoall_ref.owner(ce["op"], g, j) in mine), (g, j)
        # the landing fault of process 0 fails exactly its cell, in every process's gathered result
        f = AsResult(o["faulted"])
        want_w = [[0 if (a, b) == (0, n - 1) else 1 for b in range(n)] for a in range(n)]
        assert f.reach_write == want_w and f.reach_read == [[1] * n for _ in range(n)] and not f.aborted
        assert (f.sum_write[0][n - 1], f.xor_write[0][n - 1]) == oracle.write_checksum(SEED, 0, n - 1, f.run_seq, W)
        assert f.unreachable_pairs == 1 and not f.verdict
        h = AsResult(o["healed"])
        assert h.reach == [[1] * n for _ in range(n)] and h.verdict and h.run_seq == f.run_seq + 1
        check_full_parity(pkg, oracle, h, n, NBYTES, 1, 3)
        # a peer mapping cannot be dropped in one process of a multi-process domain (the others would not learn of
        # it), and the refusal changes nothing: the next pingpong still exchanges every pair
        assert o["unmap"] == ERR_UNSUPPORTED
        a = o["after_unmap"]
        assert a["call_seq"] == 2
        for i in mine:
            for j in range(n):
                if i != j:
                    assert a["measured"][i][j] and a["status"][i][j] == 0, (i, j)
                    assert a["digest"][i][j] == pingpong_ref.cell_digest(2, pl.partner, pl.rounds, i, j, MP_TRIPS, PP_REPS)


@pytest.mark.parametrize("world,n_local", [(2, 8), (2, 4)], ids=["2x8", "2x4"])
def test_pingpong_merges_the_status_rows_of_every_process(pkg, world, n_local):
    """Process 1's ranks are (simulated) MIG instances: they map no peer, so every pair with one of them is skipped in
    both processes, while process 0's pairs among its own ranks are exchanged.  What process 0 may exchange depends
    on process 1's status rows landing in the right rows of the merged table."""
    n = world * n_local
    outs = run_processes(world, n_local, "mig")
    pl = pkg.plan(n, NBYTES, 1)
    for rank, o in enumerate(outs):
        assert o["info"]["first"] == rank * n_local
        pp = o["pp"]
        mine = range(rank * n_local, (rank + 1) * n_local)
        for i in mine:
            for j in range(n):
                if i == j:
                    continue
                inside = rank == 0 and j < n_local
                assert pp["measured"][i][j] == inside, (rank, i, j, pp["status"][i][j])
                if inside:
                    assert pp["status"][i][j] == 0
                    assert pp["digest"][i][j] == pingpong_ref.cell_digest(1, pl.partner, pl.rounds, i, j, MP_TRIPS, PP_REPS)
                else:
                    assert pp["status"][i][j] == ERR_UNSUPPORTED, (rank, i, j, pp["status"][i][j])


@pytest.mark.parametrize("what,world,n_local", [("mismatch", 2, 2), ("oversized", 2, 9)],
                         ids=["different-n-gpus", "2x9"])
def test_inconsistent_domains_are_refused_in_every_process(pkg, what, world, n_local):
    outs = run_processes(world, n_local, what)
    assert [o["rc"] for o in outs] == [ERR_ARG] * world
