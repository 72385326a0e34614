"""One long-lived handle against an exact model (tests/handle_model.py) through seeded sequences of calls.

The daemon keeps one handle for days and interleaves periodic runs, option changes, remaps during NodePrepare /
NodeUnprepare churn, diagnoses and the on-demand measurements on it.  State that outlives a call (the loop-back pass's
counters, the phase accumulators, barrier epochs, the landing-fault descriptor, the warm-up rule, the phase tables,
the measurements' call_seq, what each landing slot holds) is only exercised by sequences, so every test here drives
one handle through many calls and compares the whole output of each call with the model:

- Run: reach bits, read and write checksums, status, run_seq, the stamp arithmetic (test_timing_gpu.check_stamps),
  the verdict restatement (verdict_ref), the traced phase kinds and peers, and `warmed`;
- Diagnose: the word_ref report of every cell, field for field, from the issuer and from the target;
- Latency: status and digest; BwCurve: bad_sizes and (S, X) per size; PingPong and Atomics: clean cells, call_seq;
- refused calls: the error code, and nothing they may not change.

A divergence fails with the seed, the step index and every step so far; the walk is generated from the seed and the
model alone, so rerunning that one test reproduces it.  Several ranks share GPU 0 (ctas 8 at most per rank, so every
rank's persistent kernel stays resident), so the file runs on one H100.  No step aborts a run, injects a watchdog
timeout or touches more than 4 GiB.
"""
import json
import random
import subprocess
import sys
import textwrap
import uuid

import pytest

import handle_model as hm
import verdict_ref
import word_ref
from conftest import ROOT, gpu_count
from test_timing_gpu import check_stamps, traces_of
from test_words_gpu import assert_report, region_offset, want_dict

pytestmark = pytest.mark.gpu

NGPU = gpu_count()
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
# bytes_per_pair is not a whole number of 16 KiB granules at any N below: the last granule is partial
BIG = (1 << 20) + 5 * 1024 + 128
SMALL = 200 * 1024 + 384
G = word_ref.GRANULE_WORDS
UNIT = 1024  # words in one 8 KiB unit of the data paths
HOPS, LAT_REPS = 64, 2
TRIPS = 16
ATOMIC_OPS = 64


class Refused(Exception):
    pass


class Driver:
    """Applies steps to a probe handle and to the model, and checks each call's output against the model."""

    def __init__(self, pkg, oracle, p, cfg, n, nbytes, me=0, nprocs=1, same_device=True):
        self.pkg, self.a, self.oracle, self.p = pkg, pkg.abi, oracle, p
        self.n, self.nbytes, self.me, self.nprocs, self.same = n, nbytes, me, nprocs, same_device
        info = p.Info()
        self.first, self.n_local = info.first_local_rank, info.n_local
        local = list(range(self.first, self.first + self.n_local))
        self.m = hm.HandleModel(oracle, hm.schedule_fn(p._lib, pkg.abi), n, nbytes, info.sm_count[0], cfg.ctas,
                                local=local, flags=cfg.flags)
        self.gate = pkg.gate(cfg, n)
        self.check_info()

    # ---- checks ----------------------------------------------------------------------------------------------
    def check_info(self):
        info = self.p.Info()
        assert [info.ctas[li] for li in range(self.n_local)] == [self.m.ctas_of(g) for g in self.m.local]
        assert info.path == self.m.path and info.bytes_per_pair == self.m.bpp

    def check_run(self, res, exp, gathered=None):
        m = self.m
        assert res.run_seq == exp["run_seq"], (res.run_seq, exp["run_seq"])
        assert not res.aborted and res.bytes_per_pair == m.bpp
        rows = [g for g in range(self.n) if (res.row_mask >> g) & 1]
        assert rows == m.local, (rows, m.local)
        for out in [res] + ([gathered] if gathered is not None else []):
            for i in [g for g in range(self.n) if (out.row_mask >> g) & 1]:
                for j in range(self.n):
                    c = exp["cells"][(i, j)]
                    got = dict(reach_read=out.reach_read[i][j], reach_write=out.reach_write[i][j],
                               read=(out.sum_read[i][j], out.xor_read[i][j]),
                               write=(out.sum_write[i][j], out.xor_write[i][j]), status=out.status[i][j])
                    want = {k: c[k] for k in got}
                    assert got == want, ("cell", i, j, got, want)
                    if c["probed"]:
                        assert out.gbps_read[i][j] > 0 and out.gbps_write[i][j] > 0, (i, j)
        traces = traces_of(self.p)
        check_stamps(res, traces)
        verdict_ref.check(res, traces, 3, m.diag, self.gate)
        for g, tr in traces.items():
            got = [{k: ph[k] for k in ("job0", "peer0", "job1", "peer1")} for ph in tr]
            assert got == m.phase_table(g), ("phase table", g, got)
        assert res.phases == len(traces[m.local[-1]])
        if exp["warmed"] is not None:
            assert res.warmed == exp["warmed"], (res.warmed, exp["warmed"])

    def check_diagnose_all(self):
        m = self.m
        for op in ("read", "write"):
            for i, j in m.cells():
                want = None
                for reader in sorted({i, j} & set(m.local)):
                    ctx = (op, i, j, reader)
                    rc, d = self.p.diagnose_raw(self.a.OP_READ if op == "read" else self.a.OP_WRITE, i, j, reader)
                    if not m.run_seq or not m.maps(reader, j):
                        assert rc == self.a.ERR_STATE, (ctx, rc)
                        continue
                    assert rc == self.a.OK, (ctx, rc)
                    if want is None:
                        spec, obs = m.diagnose(op, i, j)
                        want = want_dict(spec, obs, op, i, m.run_seq,
                                         region_offset(self.oracle, self.n, self.nbytes, 1, m.diag, op, i, j))
                    assert_report(self.pkg.Diagnosis.from_c(d), want, ctx)

    def check_cells(self, got, want, what, fields=("measured", "status")):
        for i in self.m.local:
            for j in range(self.n):
                w = want.get((i, j))
                if w is None:
                    assert not got.measured[i][j], (what, i, j)
                    continue
                for f in fields:
                    if f in w:
                        assert getattr(got, f)[i][j] == w[f], (what, f, i, j, getattr(got, f)[i][j], w[f])

    # ---- steps -----------------------------------------------------------------------------------------------
    def set_option(self, name, value):
        rc = self.p._lib.cdprobe_set_option(self.p._h, getattr(self.a, name), value)
        if rc != self.a.OK:
            raise Refused(rc)
        m = self.m
        if name == "OPT_PATH":
            m.path = value
        elif name == "OPT_CTAS":
            m.set_ctas(value)
        elif name == "OPT_CTAS_RANK":
            m.ctas[m.local[(value >> 16) - 1]] = value & 0xFFFF
        elif name == "OPT_VERIFY_CTAS":
            m.verify_ctas = value
        elif name == "OPT_WARMUP":
            m.warm_mode = value
        elif name in ("OPT_UNIDIRECTIONAL", "OPT_OVERLAP_VERIFY", "OPT_ALL_RANK_BARRIERS", "OPT_PAIR_BARRIERS"):
            m.set_flag(getattr(self.a, "FLAG" + name[3:]), bool(value))

    def apply(self, step):
        a, m, p = self.a, self.m, self.p
        kind = step[0]
        if kind == "run":
            exp = m.run()
            if self.nprocs > 1:
                raw = a.ResultT()
                assert p.run_raw(raw) == a.OK, self.pkg.abi.load_library().cdprobe_last_error()
                local = self.pkg.Result.from_c(a.ResultT.from_buffer_copy(raw))
                assert p._lib.cdprobe_gather(p._h, raw) == a.OK
                gathered = self.pkg.Result.from_c(raw)
                assert gathered.row_mask == (1 << self.n) - 1
                self.check_run(local, exp, gathered)
            else:
                self.check_run(p.Run(), exp)
        elif kind == "opt":
            self.set_option(step[1], step[2])
            self.check_info()
        elif kind == "bad_opt":  # an out-of-range value: refused, nothing changes
            before = [p.Info().ctas[li] for li in range(self.n_local)]
            with pytest.raises(Refused) as e:
                self.set_option(step[1], step[2])
            assert e.value.args[0] == a.ERR_ARG, (step, e.value.args)
            assert [p.Info().ctas[li] for li in range(self.n_local)] == before
            self.check_info()
        elif kind == "corrupt":
            _, rank, word, mask = step
            p.Corrupt(rank - self.first, 8 * word, mask)
            m.corrupt_word(rank, word, mask)
        elif kind == "landing":
            _, i, j, faults = step
            rc = p.corrupt_landing_raw(i - self.first, j, faults)
            if faults and not m.maps(i, j):
                assert rc == a.ERR_STATE, (step, rc)  # a refused arming leaves the earlier one in place
            else:
                assert rc == a.OK, (step, rc)
                m.arm(i, j, faults)
        elif kind == "unmap":
            _, i, j = step
            rc = p._lib.cdprobe_unmap_peer(p._h, i - self.first, j)
            if self.nprocs > 1:
                assert rc == a.ERR_UNSUPPORTED, rc
            else:
                assert rc == a.OK, rc
                m.unmapped.add((i, j))
        elif kind == "remap":
            _, i, j = step
            p.RemapPeer(i - self.first, j)
            m.unmapped.discard((i, j))
        elif kind == "diagnose":
            self.check_diagnose_all()
        elif kind == "latency":
            lat = p.Latency(hops=HOPS, reps=LAT_REPS)
            self.check_cells(lat, m.latency(HOPS, LAT_REPS), "latency", ("measured", "status", "digest"))
        elif kind == "pingpong":
            pp = p.PingPong(trips=TRIPS, reps=1, fenced=step[1])
            seq, want = m.pingpong()
            assert pp.call_seq == seq, (pp.call_seq, seq)
            self.check_cells(pp, want, "pingpong")
        elif kind == "atomics":
            at = p.Atomics(step[1], ops=ATOMIC_OPS, reps=1)
            seq, want = m.atomics()
            assert at.call_seq == seq, (at.call_seq, seq)
            self.check_cells(at, want, "atomics")
        elif kind == "bwcurve":
            bw = p.BwCurve(reps=1)
            seq, sizes, want = m.bwcurve()
            assert (bw.call_seq, bw.sizes, bw.path) == (seq, sizes, m.path), (bw.call_seq, seq, bw.path, m.path)
            self.check_cells(bw, want, "bwcurve", ("measured", "status", "bad_sizes"))
            for (i, j), w in want.items():
                if w["measured"]:
                    assert list(zip(bw.sum[i][j], bw.xr[i][j])) == w["sx"], ("bwcurve (S, X)", i, j)
        elif kind == "bad_call":  # refused measurement calls advance no call_seq
            what = step[1]
            if what == "bwcurve":
                rc, _ = p.bwcurve_raw(a.BWCURVE_MAX_REPS + 1)
            elif what == "pingpong":
                rc, _ = p.pingpong_raw(a.PINGPONG_MAX_TRIPS + 1, 1, 0)
            else:
                rc, _ = p.atomics_raw(3, ATOMIC_OPS, 1)
            assert rc == a.ERR_ARG, (what, rc)
        else:
            raise ValueError(step)

    def play(self, steps, label):
        """Apply `steps` in order; the first divergence fails with the label, the step index and the steps so far."""
        done = []
        for k, step in enumerate(steps):
            done.append(step)
            try:
                self.apply(step)
            except Exception as e:
                raise AssertionError(f"{label}: step {k} {step!r} diverged from the model: {e!r}\n"
                                     f"steps so far: {done!r}") from e


# ---- the seeded walk -------------------------------------------------------------------------------------------
def gen_step(rng, m, same_device=True, two_procs=False, me=0):
    """One step drawn from `rng` and the model's state alone (never from a device result)."""
    n, W = m.n, m.W
    x = rng.random()
    if x < 0.28:
        return ("run",)
    if x < 0.48:
        ctas = [1, 2, 3, 7, 8] + ([0] if n == 1 or not same_device else [])
        name, values = rng.choice([
            ("OPT_PATH", [0, 1, 2]), ("OPT_CTAS", ctas), ("OPT_VERIFY_CTAS", [1, 2, 3, 32]),
            ("OPT_UNIDIRECTIONAL", [0, 1]), ("OPT_OVERLAP_VERIFY", [0, 1]), ("OPT_ALL_RANK_BARRIERS", [0, 1]),
            ("OPT_PAIR_BARRIERS", [0, 1]), ("OPT_WARMUP", [0, 2]), ("OPT_WARMUP_BYTES", [0, 128, m.bpp + 4096]),
            ("OPT_CTAS_RANK", None)])
        if name == "OPT_CTAS_RANK":
            return ("opt", name, (rng.randrange(1, len(m.local) + 1) << 16) | rng.choice([1, 2, 3, 7, 8]))
        return ("opt", name, rng.choice(values))
    if x < 0.51:
        return ("bad_opt",) + rng.choice([("OPT_PATH", 3), ("OPT_VERIFY_CTAS", 0), ("OPT_WARMUP", 3),
                                          ("OPT_CTAS", 1 << 32), ("OPT_CTAS", (1 << 32) | 4),
                                          ("OPT_CTAS_RANK", (1 << 48) | (1 << 16) | 4),
                                          ("OPT_CTAS_RANK", ((len(m.local) + 1) << 16) | 4)])
    if x < 0.61:
        mine = [(r, k) for r, k in m.corrupt if r in m.local]
        if mine and (len(mine) >= 3 or rng.random() < 0.4):
            r, k = rng.choice(mine)
            return ("corrupt", r, k, m.corrupt[(r, k)])  # restore
        r = rng.choice(m.local)
        first = rng.randrange(m.n_slices) * W
        tail = W // G * G
        where = rng.choice([0, W - 1, rng.randrange(1, max(2, W // UNIT)) * UNIT % W,
                            tail + rng.randrange(W - tail) if W > tail else W - 1])
        return ("corrupt", r, first + where, rng.getrandbits(64) | 1 << rng.randrange(64))
    if x < 0.68:
        if m.fault and rng.random() < 0.4:
            return ("landing", m.local[0], rng.randrange(n), [])
        i = rng.choice(m.local)
        j = rng.choice([c for c in range(n) if c != i] or [i])
        words = rng.sample(sorted({0, W - 1, W // 2, rng.randrange(W), W // G * G if W % G else W - 2}), rng.randint(1, 3))
        return ("landing", i, j, [(k, rng.getrandbits(64) | 1) for k in words])
    if x < 0.75 and n > 1:
        i = rng.choice(m.local)
        down = sorted(c for c in m.unmapped if c[0] == i)
        if down and rng.random() < 0.6:
            return ("remap",) + down[0]
        j = rng.choice([c for c in range(n) if c != i])
        return ("unmap" if rng.random() < 0.7 else "remap", i, j)
    if x < 0.80:
        return ("diagnose",)
    if x < 0.85:
        return ("latency",)
    if x < 0.89:
        return ("pingpong", rng.randrange(2))
    if x < 0.94:
        return ("atomics", rng.randrange(3))
    if x < 0.98:
        return ("bwcurve",)
    return ("bad_call", rng.choice(["bwcurve", "pingpong", "atomics"]))


def walk(drv, seed, n_steps, **kw):
    rng = random.Random(seed)
    steps = []
    for k in range(n_steps):
        step = gen_step(rng, drv.m, **kw)
        steps.append(step)
        try:
            drv.apply(step)
        except Exception as e:
            raise AssertionError(f"seed {seed}: step {k} {step!r} diverged from the model: {e!r}\n"
                                 f"steps so far: {steps!r}") from e
    drv.play([("run",), ("diagnose",)], f"seed {seed}: closing run")
    return steps


def open_same(pkg, n, nbytes, ctas=8):
    cfg = pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME if n > 1 else 0, ctas=ctas, timeout_ms=20000)
    return cfg, pkg.Open(cfg)


# N = 1 opens at the full grid, a small one and the same-device grid; every walk changes the grid as it goes
WALKS = [(1, BIG, 0, 11), (1, SMALL, 3, 12), (1, BIG, 8, 13), (2, BIG, 8, 21), (2, SMALL, 8, 22), (2, BIG, 8, 23),
         (3, BIG, 8, 31), (3, SMALL, 8, 32), (3, BIG, 8, 33), (5, BIG, 8, 51), (5, SMALL, 8, 52), (5, BIG, 8, 53)]
STEPS = 60


@pytest.mark.parametrize("n,nbytes,ctas,seed", WALKS, ids=[f"n{w[0]}-{'big' if w[1] == BIG else 'small'}-seed{w[3]}"
                                                           for w in WALKS])
def test_seeded_walk(pkg, oracle, n, nbytes, ctas, seed):
    cfg, p = open_same(pkg, n, nbytes, ctas)
    with p:
        walk(Driver(pkg, oracle, p, cfg, n, nbytes), seed, STEPS)


@pytest.mark.skipif(NGPU < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("seed", [61, 62])
def test_seeded_walk_real_peers(pkg, oracle, seed):
    n = min(NGPU, 4)
    cfg = pkg.Config(ordinals=list(range(n)), bytes=BIG, timeout_ms=20000)
    with pkg.Open(cfg) as p:
        walk(Driver(pkg, oracle, p, cfg, n, BIG, same_device=False), seed, STEPS, same_device=False)


# ---- hand-written sequences: the transitions most likely to leave state behind ---------------------------------
def play(pkg, oracle, n, nbytes, steps, label, ctas=8):
    cfg, p = open_same(pkg, n, nbytes, ctas)
    with p:
        drv = Driver(pkg, oracle, p, cfg, n, nbytes)
        drv.play(steps, label)
        return drv


RUN, DIAG = ("run",), ("diagnose",)


def test_ctas_change_between_streamed_passes(pkg, oracle):
    steps = [RUN, ("opt", "OPT_CTAS", 3), RUN, DIAG, ("opt", "OPT_CTAS", 0), RUN, ("opt", "OPT_CTAS", 1), RUN, RUN,
             ("opt", "OPT_CTAS", 7), ("opt", "OPT_PATH", 1), RUN, DIAG, ("opt", "OPT_CTAS", 2), RUN]
    for nbytes in (BIG, SMALL):
        play(pkg, oracle, 1, nbytes, steps, f"n 1, {nbytes} bytes", ctas=0)


@pytest.mark.parametrize("n", [1, 2])
def test_path_change_while_a_landing_fault_is_armed(pkg, oracle, n):
    bpp = oracle.plan(n, BIG, 1, n == 1).bytes_per_pair
    j = 0 if n == 1 else 1
    faults = [(0, 1 << 63), (bpp // 8 - 1, 0xF0), (bpp // 8 // G * G + 5, 1 << 7)]
    steps = [RUN, ("landing", 0, j, faults), RUN, DIAG]
    for path in (1, 2, 0):
        steps += [("opt", "OPT_PATH", path), RUN, DIAG]
    steps += [("landing", 0, j, []), RUN, DIAG, ("opt", "OPT_PATH", 2), RUN, DIAG]
    play(pkg, oracle, n, BIG, steps, f"n {n}")


def test_unidirectional_grows_and_shrinks_the_phase_table(pkg, oracle):
    steps = [RUN]
    for uni in (1, 0, 1, 0):
        steps += [("opt", "OPT_UNIDIRECTIONAL", uni), RUN, RUN]
    steps += [("opt", "OPT_OVERLAP_VERIFY", 0), ("opt", "OPT_UNIDIRECTIONAL", 1), RUN, DIAG,
              ("opt", "OPT_UNIDIRECTIONAL", 0), RUN, ("opt", "OPT_OVERLAP_VERIFY", 1), RUN, DIAG]
    for n in (3, 5):
        play(pkg, oracle, n, BIG, steps, f"n {n}")


@pytest.mark.parametrize("n", [1, 2])
def test_measurements_between_a_corruption_and_its_restore(pkg, oracle, n):
    bpp = oracle.plan(n, BIG, 1, n == 1).bytes_per_pair
    W = bpp // 8
    word = W // G * G + 3  # inside the last, partial granule of slice 0
    steps = [("bwcurve",), ("latency",), ("corrupt", 0, word, 0xFF00), ("bwcurve",), ("latency",), RUN, DIAG,
             ("corrupt", 0, 5, 1 << 40), ("bwcurve",), ("latency",), ("corrupt", 0, word, 0xFF00), ("bwcurve",),
             ("latency",), RUN, ("corrupt", 0, 5, 1 << 40), ("bwcurve",), ("latency",), RUN, DIAG]
    play(pkg, oracle, n, BIG, steps, f"n {n}")


def test_write_cell_of_a_writer_unmapped_for_one_run(pkg, oracle):
    """The slot (0, 1) is not rewritten while the pair is down: from the target it reads STALE, one run back; the issuer
    cannot read it; after the remap the next run rewrites it.  Arming a landing fault on the unmapped cell is refused
    and leaves the earlier arming in force."""
    steps = [RUN, RUN, ("landing", 2, 0, [(5, 1 << 9)]), ("unmap", 0, 1), ("landing", 0, 1, [(3, 1)]), RUN, DIAG,
             ("landing", 0, 1, []), ("latency",), ("atomics", 0), ("pingpong", 0), ("bwcurve",),
             ("remap", 0, 1), DIAG, RUN, DIAG, ("unmap", 1, 2), RUN, RUN, DIAG, ("remap", 1, 2), RUN, DIAG]
    drv = play(pkg, oracle, 3, BIG, steps, "n 3")
    assert drv.m.slots[(0, 1)].run_seq == drv.m.run_seq


@pytest.mark.parametrize("n", [1, 2])
def test_out_of_range_ctas_are_refused(pkg, oracle, n):
    """OPT_CTAS and OPT_CTAS_RANK values whose high bits would be cut off (2^32 CTAs would become 0, a rank index
    2^32 + 1 would become rank 1): CDPROBE_ERR_ARG, Info().ctas unchanged, and the next run is at parity."""
    steps = [RUN, ("bad_opt", "OPT_CTAS", 1 << 32), RUN, ("bad_opt", "OPT_CTAS", (1 << 32) | 5),
             ("bad_opt", "OPT_CTAS_RANK", (1 << 48) | (1 << 16) | 4), RUN,
             ("bad_opt", "OPT_CTAS_RANK", (((1 << 32) + n) << 16) | 2), ("opt", "OPT_CTAS", 3), RUN, DIAG]
    play(pkg, oracle, n, BIG, steps, f"n {n}")


# ---- two processes, one rank each, on one GPU ------------------------------------------------------------------
def two_proc_steps(seed, n_steps, bpp):
    """The same list in both processes: collective steps ("all") and SetOption ("both") run in both; every other step
    belongs to one process.  Between two collective steps the processes are not ordered, so a stretch that corrupts a
    source buffer holds no step that reads another rank's memory outside a run."""
    rng = random.Random(seed)
    W = bpp // 8
    out, mutating = [], False
    while len(out) < n_steps:
        x = rng.random()
        if x < 0.35:
            out.append(("all", rng.choice([("run",), ("run",), ("pingpong", rng.randrange(2)), ("bwcurve",)])))
            mutating = rng.random() < 0.5
            continue
        if x < 0.5:
            out.append(("both", ("opt",) + rng.choice([("OPT_PATH", rng.randrange(3)), ("OPT_CTAS", rng.choice([1, 3, 8])),
                                                       ("OPT_UNIDIRECTIONAL", rng.randrange(2)),
                                                       ("OPT_OVERLAP_VERIFY", rng.randrange(2)),
                                                       ("OPT_WARMUP", rng.choice([0, 2]))])))
            continue
        owner = rng.randrange(2)
        if mutating:
            if rng.random() < 0.5:
                out.append((owner, ("corrupt", owner, rng.choice([0, W - 1, W // G * G + 1]),
                                    1 << rng.randrange(64))))
            else:
                faults = [] if rng.random() < 0.3 else [(rng.randrange(W), rng.getrandbits(64) | 1)]
                out.append((owner, ("landing", owner, 1 - owner, faults)))
        else:
            out.append((owner, rng.choice([("diagnose",), ("latency",), ("atomics", rng.randrange(3)),
                                           ("unmap", owner, 1 - owner)])))
    out.append(("all", ("run",)))
    return out


CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    sys.path.insert(0, %r)
    import cdprobe_pkg
    from oracle import oracle
    import test_handle_sequences_gpu as t
    pkg = cdprobe_pkg.load()
    session, rank, seed, nbytes = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
    cfg = pkg.Config(ordinals=[0], bytes=nbytes, world_size=2, rank=rank, session=session, flags=0x40, ctas=8,
                     timeout_ms=30000)
    with pkg.Open(cfg) as p:
        drv = t.Driver(pkg, oracle, p, cfg, 2, nbytes, me=rank, nprocs=2)
        steps = t.two_proc_steps(seed, 40, drv.m.bpp)
        done = []
        for k, (who, step) in enumerate(steps):
            done.append((who, step))
            try:
                if who in ("all", "both", rank):
                    drv.apply(step)
                else:
                    drv.mirror(step)
            except Exception as e:
                print("RESULT " + json.dumps({"ok": False, "error": f"process {rank}, seed {seed}: step {k} "
                                              f"{step!r} diverged from the model: {e!r}; steps so far: {done!r}"}))
                sys.exit(0)
    print("RESULT " + json.dumps({"ok": True, "run_seq": drv.m.run_seq, "steps": len(steps)}))
    """
) % (ROOT, ROOT + "/tests")


def mirror(self, step):
    """The model's side of a step the other process executes: its state changes, not its checks."""
    m = self.m
    kind = step[0]
    if kind == "corrupt":
        m.corrupt_word(step[1], step[2], step[3])
    elif kind == "landing":
        m.arm(step[1], step[2], step[3])


Driver.mirror = mirror


@pytest.mark.parametrize("seed", [71])
def test_two_process_sequence(pkg, oracle, seed):
    session = f"hs-{uuid.uuid4().hex[:12]}"
    procs = [subprocess.Popen([sys.executable, "-c", CHILD, session, str(r), str(seed), str(BIG)],
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for r in range(2)]
    outs = []
    for pr in procs:
        so, se = pr.communicate(timeout=600)
        assert pr.returncode == 0, se[-3000:]
        outs.append(json.loads([l for l in so.splitlines() if l.startswith("RESULT ")][-1][7:]))
    # when one process diverges the other usually fails next at a collective: report both
    assert all(o["ok"] for o in outs), [o.get("error") for o in outs]
    assert outs[0]["run_seq"] == outs[1]["run_seq"] >= hm.FIRST_RUN_SEQ
