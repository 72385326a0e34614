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
- the five all-reduces that run on one GPU (AllReduce, AllReduceTwoShot, AllReduceLL, AllReduceRing, AllReducePush):
  per row measured, status, bad_sizes and per size bad_words, first_bad and (S, X), under corruptions at rest, each
  protocol's armed faults (drop and unstored modes included), the skip rule (any down pair stops every rank) and each
  area's sticky rule; AllToAll: per rank measured and blocks, per cell status, bad_sizes and per size bad_words,
  first_bad and (S, X), under armed faults and the sticky exchange-area rule; Memcpy, both ops: per cell measured,
  status, bad_sizes and per size bad_words, first_bad and (S, X), under corruptions at rest, armed faults and the
  exchange area it shares with the all-to-all; the copy-engine all-to-all, both ops: per rank measured, status and
  blocks, per cell status, bad_sizes and per size bad_words, first_bad and (S, X) where its owner is local, under
  corruptions at rest, armed flips, drops and holds, its all-or-nothing down rule, the shared exchange area and the
  hardware-queue refusal (walks with N = 3 and 5 ranks on one device see it refused at 8 queues, and run it in a child
  process with 32); all with call_seq, the ladder and the path (the LL, the ring and the NVLS call report their own)
  or area_bytes;
- the NVLS all-reduce (AllReduceNVLS) with its fault option armed, where the domain cannot form a multicast object
  (ranks sharing a device, or one rank whose one-device object the driver refuses, asked once per process): it runs
  nothing, every row reports CDPROBE_ERR_UNSUPPORTED, its own call_seq advances, and its refusals name their reasons.
  On a domain that can form the object (the walk over real peers) the call runs the kernel, which the model does not
  cover, so no walk draws it there;
- refused calls: the error code, and nothing they may not change.

A divergence fails with the seed, the step index and every step so far; the walk is generated from the seed and the
model alone, so rerunning that one test reproduces it.  Several ranks share GPU 0 (ctas 8 at most per rank, so every
rank's persistent kernel stays resident), so the file runs on one H100.  No step aborts a run, injects a watchdog
timeout or touches more than 4 GiB.
"""
import ctypes as C
import functools
import json
import os
import random
import subprocess
import sys
import textwrap
import uuid

import pytest

import allreduce_ll_ref
import allreduce_push_ref
import allreduce_ring_ref
import bwcurve_ref
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
LADDER_REPS = 1  # the ladder measurements fold timed rep 1, the faulted one, into their (S, X)
# each ladder measurement's fault option and the model's {process: value} of it
FAULTS = {"OPT_ALLREDUCE_FAULT": "ar_fault", "OPT_ALLREDUCE_TWOSHOT_FAULT": "ts_fault",
          "OPT_ALLREDUCE_LL_FAULT": "ll_fault", "OPT_ALLREDUCE_RING_FAULT": "ring_fault",
          "OPT_ALLREDUCE_PUSH_FAULT": "push_fault", "OPT_ALLTOALL_FAULT": "a2a_fault", "OPT_MEMCPY_FAULT": "mc_fault",
          "OPT_CE_ALLTOALL_FAULT": "cea_fault", "OPT_ALLREDUCE_NVLS_FAULT": "nvls_fault"}
# each all-reduce step: the model's method, the raw binding and the path it reports (None: the handle's)
ALLREDUCES = {"allreduce": ("allreduce", "allreduce_raw", None), "twoshot": ("twoshot", "allreduce_twoshot_raw", None),
              "ll": ("ll", "allreduce_ll_raw", 3), "ring": ("ring", "allreduce_ring_raw", 4),
              "push": ("push", "allreduce_push_raw", None), "nvls": ("allreduce_nvls", "allreduce_nvls_raw", 5)}
LADDER_CALLS = [("allreduce",), ("twoshot",), ("ll",), ("ring",), ("push",), ("nvls",), ("alltoall",), ("memcpy", 1),
                ("memcpy", 2), ("ce_alltoall", 1), ("ce_alltoall", 2)]


def ladder_calls(m):
    """LADDER_CALLS without the NVLS call where it would run: the model covers it only on a domain that cannot form a
    multicast object (HandleModel.nvls_modelled)."""
    return [c for c in LADDER_CALLS if c != ("nvls",) or m.nvls_modelled()]


@functools.lru_cache(maxsize=None)
def one_device_nvls_refused(pkg, ordinal):
    """Whether a one-rank cdprobe_allreduce_nvls on `ordinal` runs nothing (CDPROBE_ERR_UNSUPPORTED): the device has no
    multicast, or its driver refuses a multicast object of one device.  Asked once, on a handle of its own."""
    with pkg.Open(pkg.Config(ordinals=[ordinal], bytes=1 << 20, ctas=8, timeout_ms=20000)) as p:
        ar = p.AllReduceNVLS(reps=1)
    assert ar.measured[0] or ar.status[0] == hm.ERR_UNSUPPORTED, ar.status
    return not ar.measured[0]


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
        # every process of these tests opens its ranks on the same ordinals, so global rank g sits on ordinal
        # cfg.ordinals[g % n_local] (the copy-engine all-to-all counts hardware queues per device)
        self.m.ordinal.update({g: cfg.ordinals[g % self.n_local] for g in range(n)})
        if n == 1:
            self.m.one_device_nvls_refused = one_device_nvls_refused(pkg, cfg.ordinals[0])
        self.gate = pkg.gate(cfg, n)
        self.area_bytes = None  # of the exchange area, once the all-to-all or memcpy has reported it
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

    def table_fits(self, name, value):
        """Whether cdprobe_schedule accepts every local rank's table with schedule option `name` set to `value`
        (UNIDIRECTIONAL with the serial verify overflows the phase table from N = 13)."""
        if name not in ("OPT_UNIDIRECTIONAL", "OPT_OVERLAP_VERIFY", "OPT_ALL_RANK_BARRIERS", "OPT_PAIR_BARRIERS"):
            return True
        m, flag = self.m, getattr(self.a, "FLAG" + name[3:])
        flags = (m.flags & ~flag) | (flag if value else 0)
        flags = flags if flags & hm.FLAG_OVERLAP_VERIFY else flags | hm.FLAG_SERIAL_VERIFY
        s = self.a.ScheduleT()
        return all(self.p._lib.cdprobe_schedule(self.n, g, self.nbytes, m.mode, m.ops, flags, m.ctas_of(g),
                                                m.verify_ctas, C.byref(s)) == 0 for g in m.local)

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
        elif name in FAULTS:
            m.arm_measure(getattr(m, FAULTS[name]), self.me, value)

    def check_allreduce(self, kind="allreduce"):
        a, m = self.a, self.m
        model, raw, path = ALLREDUCES[kind]
        want = getattr(m, model)(LADDER_REPS, proc=self.me) if kind == "nvls" else getattr(m, model)(LADDER_REPS)
        rc, t = getattr(self.p, raw)(LADDER_REPS)
        if want is None or isinstance(want, str):  # the armed fault names nothing of the ladder: refused, nothing
            assert rc == a.ERR_ARG and t.call_seq == 0 and sum(t.measured) == 0, (rc, t.call_seq)  # advances
            if isinstance(want, str):  # the NVLS call's refusal names its reason
                assert self.p._lib.cdprobe_last_error().decode() == want
            return
        assert rc == a.OK, rc
        ar = self.pkg.AllReduce.from_c(t)
        path = m.path if path is None else path
        assert (ar.call_seq, ar.sizes, ar.path, ar.reps) == (want["call_seq"], want["sizes"], path, LADDER_REPS), \
            (ar.call_seq, want["call_seq"], ar.path, path)
        assert ar.row_mask == sum(1 << g for g in m.local)
        for g, w in want["rows"].items():
            got = dict(measured=ar.measured[g], status=ar.status[g])
            if w["measured"]:
                got.update(bad_sizes=ar.bad_sizes[g], sx=list(zip(ar.sum[g], ar.xr[g])), bad_words=ar.bad_words[g],
                           first_bad=ar.first_bad[g])
            assert got == w, ("allreduce row", g, got, w)

    def check_alltoall(self):
        a, m = self.a, self.m
        want = m.alltoall(LADDER_REPS)
        rc, t = self.p.alltoall_raw(LADDER_REPS)
        if want is None:  # the armed fault names no cell, size or word of the ladder: refused, nothing advances
            assert rc == a.ERR_ARG and t.call_seq == 0 and sum(t.measured) == 0, (rc, t.call_seq)
            return
        assert rc == a.OK, rc
        aa = self.pkg.AllToAll.from_c(t)
        assert (aa.call_seq, aa.sizes, aa.path, aa.reps) == (want["call_seq"], want["sizes"], m.path, LADDER_REPS), \
            (aa.call_seq, want["call_seq"], aa.path, m.path)
        assert aa.area_bytes == (self.n * m.bpp + (2 << 20) - 1) // (2 << 20) * (2 << 20)
        self.check_area_bytes(aa.area_bytes)
        for g, w in want["ranks"].items():
            assert aa.measured[g] == w["measured"], ("alltoall rank", g)
            if w["measured"]:
                assert aa.status[g] == 0 and aa.blocks[g] == w["blocks"], ("alltoall rank", g, aa.blocks[g], w)
        for s in range(self.n):
            for d in m.local:
                w = want["cells"].get((s, d), dict(cell_measured=False, cell_status=0))
                got = dict(cell_measured=aa.cell_measured[s][d], cell_status=aa.cell_status[s][d])
                if w["cell_measured"]:
                    got.update(bad_sizes=aa.bad_sizes[s][d], bad_words=aa.bad_words[s][d],
                               first_bad=aa.first_bad[s][d], sx=list(zip(aa.sum[s][d], aa.xr[s][d])))
                assert got == w, ("alltoall cell", s, d, got, w)

    def check_area_bytes(self, area_bytes):
        """The all-to-all and memcpy share one exchange area: every call reports the same size, n blocks at least."""
        if self.area_bytes is None:
            assert area_bytes >= self.n * self.m.bpp, (area_bytes, self.n * self.m.bpp)
            self.area_bytes = area_bytes
        assert area_bytes == self.area_bytes, (area_bytes, self.area_bytes)

    def check_memcpy(self, op):
        a, m = self.a, self.m
        want = m.memcpy(op, LADDER_REPS)
        rc, t = self.p.memcpy_raw(op, LADDER_REPS)
        if want is None:  # the op or the armed fault names nothing of this call: refused, nothing advances
            assert rc == a.ERR_ARG and t.call_seq == 0 and sum(t.measured) == 0, (rc, t.call_seq)
            return
        assert rc == a.OK, rc
        mc = self.pkg.Memcpy.from_c(t)
        assert (mc.call_seq, mc.sizes, mc.op, mc.reps) == (want["call_seq"], want["sizes"], op, LADDER_REPS), \
            (mc.call_seq, want["call_seq"])
        self.check_area_bytes(mc.area_bytes)
        assert mc.row_mask == sum(1 << g for g in m.local)
        for g in m.local:
            for j in range(self.n):
                w = want["cells"].get((g, j), dict(measured=False, status=0))
                got = dict(measured=mc.measured[g][j], status=mc.status[g][j])
                assert got == {f: w[f] for f in got}, ("memcpy cell", op, g, j, got, w)
                if w["measured"]:
                    got.update(bad_sizes=mc.bad_sizes[g][j], sx=list(zip(mc.sum[g][j], mc.xr[g][j])),
                               bad_words=mc.bad_words[g][j], first_bad=mc.first_bad[g][j])
                assert got == w, ("memcpy cell", op, g, j, got, w)

    def check_ce_alltoall(self, op):
        """cdprobe_ce_alltoall against the model, field for field but the times: a refusal's code and nothing advanced;
        else call_seq, the ladder, area_bytes, per rank measured, status and blocks, and per cell cell_measured,
        cell_status and, where a local owner checked it, bad_sizes and per size bad_words, first_bad and (S, X)."""
        a, m = self.a, self.m
        want = m.ce_alltoall(op, LADDER_REPS)
        rc, t = self.p.ce_alltoall_raw(op, LADDER_REPS)
        if not isinstance(want, dict):  # ERR_ARG or the queue refusal: nothing advances, the area is not built
            assert rc == want and t.call_seq == 0 and sum(t.measured) == 0, (rc, want, t.call_seq)
            return
        assert rc == a.OK, (rc, a.load_library().cdprobe_last_error())
        ca = self.pkg.CeAllToAll.from_c(t)
        assert (ca.call_seq, ca.sizes, ca.op, ca.reps) == (want["call_seq"], want["sizes"], op, LADDER_REPS), \
            (ca.call_seq, want["call_seq"])
        assert ca.area_bytes >= want["area_min_bytes"], (ca.area_bytes, want["area_min_bytes"])
        self.check_area_bytes(ca.area_bytes)
        assert ca.row_mask == sum(1 << g for g in m.local)
        for g in range(self.n):
            w = want["ranks"].get(g, dict(measured=False, status=0, blocks=0))
            got = dict(measured=ca.measured[g], status=ca.status[g], blocks=ca.blocks[g] if ca.measured[g] else 0)
            assert got == w, ("ce_alltoall rank", op, g, got, w)
        for g in range(self.n):
            for j in range(self.n):
                w = want["cells"].get((g, j), dict(cell_measured=False, cell_status=0))
                got = dict(cell_measured=ca.cell_measured[g][j], cell_status=ca.cell_status[g][j])
                if w["cell_measured"]:
                    got.update(bad_sizes=ca.bad_sizes[g][j], bad_words=ca.bad_words[g][j],
                               first_bad=ca.first_bad[g][j], sx=list(zip(ca.sum[g][j], ca.xr[g][j])))
                assert got == w, ("ce_alltoall cell", op, g, j, got, w)

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
            if self.table_fits(step[1], step[2]):
                self.set_option(step[1], step[2])
            else:  # the schedule has no room for the phase table these flags ask for: refused, nothing changes
                with pytest.raises(Refused) as e:
                    self.set_option(step[1], step[2])
                assert e.value.args[0] == a.ERR_ARG, (step, e.value.args)
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
        elif kind in ALLREDUCES:
            self.check_allreduce(kind)
        elif kind == "alltoall":
            self.check_alltoall()
        elif kind == "memcpy":
            self.check_memcpy(step[1])
        elif kind == "ce_alltoall":
            self.check_ce_alltoall(step[1])
        elif kind == "bad_call":  # refused measurement calls advance no call_seq
            what = step[1]
            if what == "bwcurve":
                rc, _ = p.bwcurve_raw(a.BWCURVE_MAX_REPS + 1)
            elif what in ALLREDUCES:
                rc, _ = getattr(p, ALLREDUCES[what][1])(a.ALLREDUCE_MAX_REPS + 1)
            elif what == "memcpy":
                rc, _ = p.memcpy_raw(a.OP_READ | a.OP_WRITE, 1)
            elif what == "memcpy_reps":
                rc, _ = p.memcpy_raw(a.OP_WRITE, a.MEMCPY_MAX_REPS + 1)
            elif what == "alltoall":
                rc, _ = p.alltoall_raw(a.ALLTOALL_MAX_REPS + 1)
            elif what == "ce_alltoall":
                rc, t = p.ce_alltoall_raw(a.OP_READ | a.OP_WRITE, 1)
                assert t.call_seq == 0
            elif what == "ce_alltoall_reps":
                rc, t = p.ce_alltoall_raw(a.OP_WRITE, 65)
                assert t.call_seq == 0
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
def edge_word(rng, size):
    """A word of the first `size` bytes where the ladder kernels go wrong: word 0, the last word, or a word of the last
    partial 8 KiB unit (of the last unit when it is whole)."""
    words = size // 8
    lo = size // (UNIT * 8) * UNIT if size % (UNIT * 8) else words - UNIT
    return rng.choice([0, words - 1, rng.randrange(lo, words)])


def ladder_fault(rng, m, name, rank, peer):
    """A valid value of a ladder measurement's fault option at an edge word of a size of its ladder (the last size or a
    random one), acting in the process that hosts `rank`, about half of them in a drop or unstored mode:
    OPT_ALLREDUCE_FAULT on `rank`, adding 1 or dropping the word's unit; OPT_ALLREDUCE_TWOSHOT_FAULT to receiver
    `rank`, xor 1 or drop; OPT_ALLREDUCE_LL_FAULT, a corrupted packet rank -> peer, or a word `rank` never stores;
    OPT_ALLREDUCE_RING_FAULT, a corrupted or dropped push by `rank` in a phase that pushes the word (at N = 1, where
    nothing is pushed, a 5 us delay); OPT_ALLREDUCE_PUSH_FAULT, modes 0-2 by sender `rank` or mode 3 to receiver
    `rank`; OPT_ALLREDUCE_NVLS_FAULT, xor 1 or a skipped unit, by the word's owner; OPT_ALLTOALL_FAULT on block
    rank -> peer; OPT_MEMCPY_FAULT on cell rank -> peer, flipped or dropped;
    OPT_CE_ALLTOALL_FAULT on cell rank -> peer, flipped, dropped or held."""
    n = m.n
    sizes = allreduce_ll_ref.ladder(m.bpp) if name == "OPT_ALLREDUCE_LL_FAULT" else bwcurve_ref.ladder(m.bpp)
    k = rng.choice([len(sizes) - 1, rng.randrange(len(sizes))])
    word = edge_word(rng, sizes[k])
    low = ((k + 1) << 24) | word
    drop = rng.randrange(2)
    if name in ("OPT_ALLREDUCE_FAULT", "OPT_ALLREDUCE_TWOSHOT_FAULT"):
        return (drop << 48) | ((rank + 1) << 32) | low
    if name == "OPT_ALLREDUCE_LL_FAULT":
        if drop or peer == rank:
            return (2 << 48) | ((rank + 1) << 40) | ((rank + 1) << 32) | low
        return ((rank + 1) << 40) | ((peer + 1) << 32) | low
    if name == "OPT_ALLREDUCE_RING_FAULT":
        if n == 1:
            return (2 << 48) | (1 << 32) | ((k + 1) << 24) | 5
        # `rank` pushes every chunk but its own in the reduce-scatter and every chunk but rank + 1's in the all-gather,
        # so at N >= 2 one of the phases pushes the word's chunk
        phase = rng.randrange(2)
        if allreduce_ring_ref.chunk_of(sizes[k], n, word) not in allreduce_ring_ref.pushes(n, rank, phase):
            phase ^= 1
        return (drop << 48) | (phase << 40) | ((rank + 1) << 32) | low
    if name == "OPT_ALLREDUCE_PUSH_FAULT":
        mode = rng.randrange(4)
        if mode == 3 and (n == 1 or allreduce_push_ref.word_owner(sizes[k], n, word) == rank):
            mode = rng.randrange(3)
        return (mode << 48) | ((rank + 1) << 32) | low
    if name == "OPT_ALLREDUCE_NVLS_FAULT":  # no rank field: the word's owner acts on it
        return (drop << 48) | low
    if name == "OPT_MEMCPY_FAULT":
        return (drop << 48) | ((rank + 1) << 40) | ((peer + 1) << 32) | low
    if name == "OPT_CE_ALLTOALL_FAULT":  # a flip, a dropped copy, or a hold of at most 1 ms
        mode = rng.randrange(3)
        arg = rng.choice([50, 1000]) if mode == 2 else word
        return (mode << 48) | ((rank + 1) << 40) | ((peer + 1) << 32) | ((k + 1) << 24) | arg
    return ((rank + 1) << 40) | ((peer + 1) << 32) | low


def past_its_size(m, name, value):
    """The same fault one word past its size, which the next call refuses (a delay is left as it is)."""
    if name in ("OPT_ALLREDUCE_RING_FAULT", "OPT_CE_ALLTOALL_FAULT") and value >> 48 == 2:
        return value
    return value + bwcurve_ref.ladder(m.bpp)[((value >> 24) & 0xFF) - 1] // 8 - (value & 0xFFFFFF)


def gen_step(rng, m, same_device=True, two_procs=False, me=0, ctas_cap=None):
    """One step drawn from `rng` and the model's state alone (never from a device result).  `ctas_cap` bounds the
    grids it may ask for, so that many same-device ranks stay resident together.  A sixth of the steps are calls of the
    ladder collectives (the six all-reduces where ladder_calls keeps the NVLS call, the all-to-all, memcpy and the
    copy-engine all-to-all with either op, each about as often as
    bwcurve) and their fault armings; the rest keep their weights."""
    n, W = m.n, m.W
    grids = [c for c in (1, 2, 3, 7, 8) if ctas_cap is None or c <= ctas_cap]
    x = rng.random()
    if x < 0.12:
        return rng.choice(ladder_calls(m))
    if x < 0.16:
        name = rng.choice(sorted(FAULTS))
        if getattr(m, FAULTS[name]) and rng.random() < 0.4:
            return ("opt", name, 0)
        i = rng.choice(m.local)
        j = rng.choice([c for c in range(n) if c != i] or [i])
        value = ladder_fault(rng, m, name, i, j)
        if rng.random() < 0.15:  # one word past its size: the next call is refused until the fault is re-armed
            value = past_its_size(m, name, value)
        elif name == "OPT_ALLREDUCE_NVLS_FAULT" and rng.random() < 0.1:  # a mode above 1, or bits that name nothing
            value |= rng.choice([2 << 48, 1 << 32])
        return ("opt", name, value)
    x = (x - 0.16) / 0.84
    if x < 0.28:
        return ("run",)
    if x < 0.48:
        ctas = grids + ([0] if n == 1 or not same_device else [])
        name, values = rng.choice([
            ("OPT_PATH", [0, 1, 2]), ("OPT_CTAS", ctas), ("OPT_VERIFY_CTAS", [1, 2, 3, 32]),
            ("OPT_UNIDIRECTIONAL", [0, 1]), ("OPT_OVERLAP_VERIFY", [0, 1]), ("OPT_ALL_RANK_BARRIERS", [0, 1]),
            ("OPT_PAIR_BARRIERS", [0, 1]), ("OPT_WARMUP", [0, 2]), ("OPT_WARMUP_BYTES", [0, 128, m.bpp + 4096]),
            ("OPT_CTAS_RANK", None)])
        if name == "OPT_CTAS_RANK":
            return ("opt", name, (rng.randrange(1, len(m.local) + 1) << 16) | rng.choice(grids))
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
    return ("bad_call", rng.choice(["bwcurve", "pingpong", "atomics", "alltoall", "memcpy", "memcpy_reps", "ce_alltoall",
                                    "ce_alltoall_reps"] + sorted(ALLREDUCES)))


def walk_step(rng, m, steps, **kw):
    """The next step of a walk: right after an unmap or a remap, a call of one of the ladder collectives (ladder_calls), so that
    every walk with churn calls them while a pair is down and after a remap; else gen_step's."""
    if steps and steps[-1][0] in ("unmap", "remap"):
        return rng.choice(ladder_calls(m))
    return gen_step(rng, m, **kw)


def walk(drv, seed, n_steps, **kw):
    rng = random.Random(seed)
    steps = []
    for k in range(n_steps):
        step = walk_step(rng, drv.m, steps, **kw)
        steps.append(step)
        try:
            drv.apply(step)
        except Exception as e:
            raise AssertionError(f"seed {seed}: step {k} {step!r} diverged from the model: {e!r}\n"
                                 f"steps so far: {steps!r}") from e
    # remap what is still down, so that every walk with churn also calls the ladder measurements after a remap
    closing = [("remap",) + c for c in sorted(drv.m.unmapped)] + ladder_calls(drv.m) + [("run",), ("diagnose",)]
    drv.play(closing, f"seed {seed}: closing run")
    return steps + closing


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


# The copy-engine all-to-all needs n x n hardware queues for n ranks on one device: above 2 ranks more than the
# default 8 of CUDA_DEVICE_MAX_CONNECTIONS, so the walks above see its refusal at N = 3 and 5, and these see it run.
# The CUDA runtime reads the variable once, at its start, so they run in a child process that has it from birth.
CHILD_WALKS = [(3, BIG, 8, 34), (5, SMALL, 8, 54)]


def case_walk(pkg, oracle, n, nbytes, ctas, seed):
    cfg, p = open_same(pkg, n, nbytes, ctas)
    with p:
        drv = Driver(pkg, oracle, p, cfg, n, nbytes)
        assert drv.m.max_connections == {0: 32}
        walk(drv, seed, STEPS)


@pytest.mark.parametrize("n,nbytes,ctas,seed", CHILD_WALKS,
                         ids=[f"n{w[0]}-{'big' if w[1] == BIG else 'small'}-seed{w[3]}" for w in CHILD_WALKS])
def test_seeded_walk_with_32_hardware_queues(pkg, oracle, n, nbytes, ctas, seed):
    in_child("case_walk", n, nbytes, ctas, seed)


SEQ_CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path[:0] = [%r, %r]
    sys.modules["torch"] = None  # not needed here; conftest.gpu_count() then reports 0, which only feeds skip marks
    import cdprobe_pkg
    from oracle import oracle
    import test_handle_sequences_gpu as t
    pkg = cdprobe_pkg.load()
    getattr(t, sys.argv[1])(pkg, oracle, *json.loads(sys.argv[2]))
    print("CHILD OK")
    """
) % (ROOT, ROOT + "/tests")


def in_child(case, *args, timeout=1200):
    """Run case(pkg, oracle, *args) in a fresh process with 32 hardware queues per device; its assertion is the
    failure message."""
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    pr = subprocess.run([sys.executable, "-c", SEQ_CHILD, case, json.dumps(args)], env=env, capture_output=True,
                        text=True, timeout=timeout)
    assert pr.returncode == 0 and "CHILD OK" in pr.stdout, pr.stderr[-8000:]


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
    AR, A2A = ("allreduce",), ("alltoall",)
    steps = [("bwcurve",), ("latency",), AR, ("corrupt", 0, word, 0xFF00), ("bwcurve",), ("latency",), AR, A2A, RUN,
             DIAG, ("corrupt", 0, 5, 1 << 40), ("bwcurve",), ("latency",), AR, ("corrupt", n - 1, 5, 1 << 41), AR,
             ("corrupt", 0, word, 0xFF00), ("bwcurve",), ("latency",), AR, RUN, ("corrupt", 0, 5, 1 << 40),
             ("corrupt", n - 1, 5, 1 << 41), ("bwcurve",), ("latency",), AR, A2A, RUN, DIAG]
    play(pkg, oracle, n, BIG, steps, f"n {n}")


def test_alltoall_area_of_a_pair_unmapped_at_its_first_call_stays_unmapped_after_the_remap(pkg, oracle):
    """The exchange area is mapped at the first all-to-all only where the probe mapping is up, and remaps leave it
    alone: cell (0, 2) is skipped before and after its remap, until close, while runs use the remapped pair.  The
    all-to-all leaves the landing slots as the last run wrote them."""
    A2A = ("alltoall",)
    steps = [RUN, ("unmap", 0, 2), A2A, ("allreduce",), ("remap", 0, 2), A2A, RUN, DIAG, A2A, DIAG,
             ("opt", "OPT_ALLTOALL_FAULT", (3 << 40) | (1 << 32) | (1 << 24)), A2A, ("allreduce",), RUN, DIAG]
    drv = play(pkg, oracle, 3, BIG, steps, "n 3")
    assert drv.m.area_down == {(0, 2)} and drv.m.a2a_calls == 4


def case_exchange_area_built_while_a_pair_is_down(pkg, oracle, first):
    """cdprobe_memcpy, cdprobe_alltoall and cdprobe_ce_alltoall share one exchange area, built by whichever is called
    first, even by a copy-engine all-to-all that then runs nothing: with (0, 2) down then, cell (0, 2) is skipped by
    memcpy and the all-to-all, with either op, until close, while runs use the remapped pair, and the copy-engine
    all-to-all stays off.  An armed memcpy drop on another cell fails exactly that cell and size, and the next call is
    clean again.  Three ranks on one device need 9 hardware queues: it runs in a child process with 32."""
    A2A, MC1, MC2, CE1, CE2 = ("alltoall",), ("memcpy", 1), ("memcpy", 2), ("ce_alltoall", 1), ("ce_alltoall", 2)
    opener = {"memcpy": MC1, "alltoall": A2A, "ce_alltoall": CE1}[first]
    bpp = oracle.plan(3, BIG, 1, False).bytes_per_pair
    last = len(bwcurve_ref.ladder(bpp)) - 1
    drop = (1 << 48) | (3 << 40) | (1 << 32) | ((last + 1) << 24) | (bpp // 8 - 1)
    # the first calls after the remap are memcpy's, so a model that let only the all-to-all build the area diverges
    # (a copy-engine all-to-all that runs nothing is the only call before the remap, so a library that built the area
    # after its down check would build it at the next memcpy, with every pair up)
    steps = [RUN, ("unmap", 0, 2), opener] + ([MC2] if first != "ce_alltoall" else []) + [
        ("remap", 0, 2), MC1, MC2, A2A, CE2, RUN, DIAG, ("opt", "OPT_MEMCPY_FAULT", drop), MC2, MC1,
        ("opt", "OPT_MEMCPY_FAULT", 0), MC2, A2A, CE1, RUN, DIAG]
    drv = play(pkg, oracle, 3, BIG, steps, f"n 3, {first} first")
    assert drv.m.max_connections == {0: 32}
    assert drv.m.area_down == {(0, 2)}
    assert (drv.m.mc_calls, drv.m.cea_calls) == {"memcpy": (7, 2), "alltoall": (6, 2), "ce_alltoall": (5, 3)}[first]


@pytest.mark.parametrize("first", ["memcpy", "alltoall", "ce_alltoall"])
def test_exchange_area_built_while_a_pair_is_down_stays_unmapped_for_memcpy_and_alltoall(pkg, oracle, first):
    in_child("case_exchange_area_built_while_a_pair_is_down", first)


def allreduce_edge_faults(m, drop):
    """One armed fault per all-reduce at an edge word (word 0 of size 0, or the last word of the last, partial unit),
    in its drop or unstored mode when `drop`, else as a corrupted word; each in a rank of this process."""
    n, W = m.n, m.W
    sizes, ll_sizes = bwcurve_ref.ladder(m.bpp), allreduce_ll_ref.ladder(m.bpp)
    last, ll_last = len(sizes) - 1, len(ll_sizes) - 1
    r, q = n - 1, 0
    out = [("OPT_ALLREDUCE_FAULT", (drop << 48) | ((r + 1) << 32) | ((last + 1) << 24) | (W - 1)),
           ("OPT_ALLREDUCE_TWOSHOT_FAULT", (drop << 48) | ((q + 1) << 32) | (1 << 24)),
           ("OPT_ALLREDUCE_LL_FAULT", (2 << 48) | ((r + 1) << 40) | ((r + 1) << 32) | ((ll_last + 1) << 24)
            | (ll_sizes[-1] // 8 - 1) if drop or n == 1 else ((r + 1) << 40) | ((q + 1) << 32) | (1 << 24)),
           ("OPT_ALLREDUCE_PUSH_FAULT", ((1 if drop else 0) << 48) | ((r + 1) << 32) | ((last + 1) << 24) | (W - 1))]
    if n > 1:  # the ring pushes the last word in the reduce-scatter from every rank but its chunk's owner, n - 1
        out.append(("OPT_ALLREDUCE_RING_FAULT", (drop << 48) | ((q + 1) << 32) | ((last + 1) << 24) | (W - 1)))
    return out


@pytest.mark.parametrize("n", [1, 3])
def test_five_allreduces_in_sequence_leave_nothing_another_could_hide_behind(pkg, oracle, n):
    """The one-shot, two-shot, LL, ring and push, one after another in both orders, on every path and across grid
    changes, between a corruption and its restore, with each one's fault armed once at an edge word, as a drop, an
    unstored word or a corrupted one.  Each rep's check clears the output it read, so a unit one of them drops reads
    as 0s rather than as the sums an earlier rep or call stored there.  (None of these calls leaves a correct sum in
    the scratch for the next: what stays there is cleared output or granule tables, so the host's zeroing of the
    LL's output at the start of a call is seen only through a memcpy diagnosis, in the test below.)"""
    FIVE = [("allreduce",), ("twoshot",), ("ll",), ("ring",), ("push",)]
    cfg, p = open_same(pkg, n, SMALL, 8)
    with p:
        drv = Driver(pkg, oracle, p, cfg, n, SMALL)
        m = drv.m
        word = m.W - 1  # in the last, partial unit of slice 0
        grids = [("OPT_CTAS", 1), ("OPT_CTAS", 3), ("OPT_CTAS_RANK", (len(m.local) << 16) | 2), ("OPT_CTAS", 8)]
        steps = []
        for q, path in enumerate((0, 1, 2)):
            steps += [("opt", "OPT_PATH", path), ("opt",) + grids[q]] + FIVE + [("corrupt", n - 1, word, 1 << 21)]
            steps += FIVE[::-1]
            for drop in (1, 0):
                faults = allreduce_edge_faults(m, drop)
                steps += [("opt",) + f for f in faults] + FIVE + [("opt",) + grids[q + 1]] + FIVE[::-1]
                steps += [("opt", f[0], 0) for f in faults]
            steps += [("corrupt", n - 1, word, 1 << 21)] + FIVE
        steps += [RUN, DIAG]
        drv.play(steps, f"n {n}")
        assert (m.ar_calls, m.ts_calls, m.ll_calls, m.ring_calls, m.push_calls) == (21,) * 5


# The LL's output lies at kArOutOff = 63232 bytes into the rank's scratch, and memcpy's last diagnosis (a DiagOut at
# 62976) leaves its first sample's `expected`, the pattern word of the lowest bad word, at 63568: over output word 42.
# At N = 1 that pattern word is the LL's sum for the word.  Each later sample's `expected` lies 48 bytes (6 words) on.
LL_WORDS_UNDER_DIAG_SAMPLES = [42 + 6 * i for i in range(16)]


@pytest.mark.parametrize("op", [1, 2], ids=["pull", "push"])
def test_an_ll_word_never_stored_is_not_hidden_by_a_memcpy_diagnosis_left_in_the_scratch(pkg, oracle, op):
    """A memcpy over corrupted source words leaves, in the scratch the LL writes its output to, the samples of its last
    diagnosis: at N = 1 their `expected` words are the LL's correct sums for the very words they lie over.  An LL that
    then never stores one of those words (mode 2) must still find it bad: the output is zeroed at the start of every LL
    call, so the word reads 0 rather than the leftover.  A clean LL first grows the scratch to the LL's size, so the
    memcpy and the faulted LL use the same buffer."""
    words = LL_WORDS_UNDER_DIAG_SAMPLES
    corrupt = [("corrupt", 0, w, 1 << 12) for w in words]
    steps = [("ll",)]
    for w in (words[0], words[-1]):
        steps += corrupt + [("memcpy", op)] + corrupt  # the corruptions are restored before the LL runs
        steps += [("opt", "OPT_ALLREDUCE_LL_FAULT", (2 << 48) | (1 << 40) | (1 << 32) | (1 << 24) | w), ("ll",),
                  ("opt", "OPT_ALLREDUCE_LL_FAULT", 0), ("ll",)]
    drv = play(pkg, oracle, 1, SMALL, steps, f"n 1, op {op}")
    assert drv.m.ll_calls == 5 and drv.m.corrupt == {}


@pytest.mark.parametrize("n", [1, 3])
def test_memcpy_leaves_the_probe_state_alone(pkg, oracle, n):
    """Memcpy copies into the exchange area and checks in the issuers' scratch: every landing slot and source checksum
    stays as the runs and corruptions left them, and a corrupted source word fails exactly the cells that copy it."""
    bpp = oracle.plan(n, BIG, 1, n == 1).bytes_per_pair
    W, j = bpp // 8, (1 if n > 1 else 0)
    faults = [(0, 1 << 63), (W - 1, 0xF0)]
    steps = [RUN, ("memcpy", 1), DIAG, ("landing", 0, j, faults), RUN, ("memcpy", 2), DIAG,
             ("corrupt", n - 1, W - 1, 1 << 30), ("memcpy", 1), ("memcpy", 2), RUN, DIAG, ("landing", 0, j, []),
             ("memcpy", 2), ("corrupt", n - 1, W - 1, 1 << 30), RUN, ("memcpy", 1), DIAG]
    play(pkg, oracle, n, BIG, steps, f"n {n}")


@pytest.mark.parametrize("n", [1, 3])
def test_grid_and_path_changes_between_ladder_calls_with_faults_armed(pkg, oracle, n):
    """OPT_CTAS and OPT_CTAS_RANK change the grid the all-reduce and the all-to-all launch on, and with it which warp
    walks which unit and stores the armed fault's word: on every path, with a fault armed on each, at an edge word."""
    bpp = oracle.plan(n, SMALL, 1, n == 1).bytes_per_pair
    sizes = bwcurve_ref.ladder(bpp)
    last, W = len(sizes) - 1, bpp // 8
    j = (n - 1) % n if n > 1 else 0
    partial = W // UNIT * UNIT + 1  # in the last, partial unit of the last size
    ar = [((n - 1 + 1) << 32) | ((last + 1) << 24) | (W - 1), (1 << 32) | (1 << 24) | 0]
    a2a = [(1 << 40) | ((j + 1) << 32) | ((last + 1) << 24) | partial,
           ((n - 1 + 1) << 40) | (1 << 32) | (1 << 24) | (sizes[0] // 8 - 1)]
    grids = [("OPT_CTAS", 1), ("OPT_CTAS", 3), ("OPT_CTAS_RANK", (1 << 16) | 7), ("OPT_CTAS", 2),
             ("OPT_CTAS_RANK", (n << 16) | 1), ("OPT_CTAS", 8)]
    steps = []
    for path in (0, 1, 2):
        steps += [("opt", "OPT_PATH", path)]
        for q, grid in enumerate(grids):
            steps += [("opt", "OPT_ALLREDUCE_FAULT", ar[q % 2]), ("opt", "OPT_ALLTOALL_FAULT", a2a[q % 2]),
                      ("allreduce",), ("alltoall",), ("opt",) + grid, ("allreduce",), ("alltoall",)]
    steps += [("opt", "OPT_ALLREDUCE_FAULT", 0), ("opt", "OPT_ALLTOALL_FAULT", 0), ("allreduce",), ("alltoall",), RUN,
              DIAG]
    play(pkg, oracle, n, SMALL, steps, f"n {n}")


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
def two_proc_steps(seed, n_steps, m):
    """The same list in both processes: collective steps ("all") and SetOption ("both") run in both; every other step
    belongs to one process.  Between two collective steps the processes are not ordered, so a stretch that corrupts a
    source buffer holds no step that reads another rank's memory outside a run."""
    rng = random.Random(seed)
    W = m.W
    out, mutating = [], False
    while len(out) < n_steps:
        x = rng.random()
        if x < 0.35:
            out.append(("all", rng.choice([("run",), ("run",), ("pingpong", rng.randrange(2)), ("bwcurve",)]
                                          + ladder_calls(m))))
            mutating = rng.random() < 0.5
            continue
        if x < 0.5:
            out.append(("both", ("opt",) + rng.choice([("OPT_PATH", rng.randrange(3)), ("OPT_CTAS", rng.choice([1, 3, 8])),
                                                       ("OPT_UNIDIRECTIONAL", rng.randrange(2)),
                                                       ("OPT_OVERLAP_VERIFY", rng.randrange(2)),
                                                       ("OPT_WARMUP", rng.choice([0, 2]))])))
            continue
        owner = rng.randrange(2)
        if x < 0.58:  # a valid fault armed (or disarmed) only by the process that hosts its rank, sender or issuer
            name = rng.choice(sorted(FAULTS))
            if name == "OPT_ALLREDUCE_RING_FAULT":
                owner = 0  # one process arms the ring, so no two of its pushes are faulted in one rep
            value = 0 if rng.random() < 0.3 else ladder_fault(rng, m, name, owner, 1 - owner)
            out.append((owner, ("opt", name, value)))
            continue
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
        steps = t.two_proc_steps(seed, 40, drv.m)
        done = []
        for k, (who, step) in enumerate(steps):
            done.append((who, step))
            try:
                if who in ("all", "both", rank):
                    drv.apply(step)
                else:
                    drv.mirror(step, who)
            except Exception as e:
                print("RESULT " + json.dumps({"ok": False, "error": f"process {rank}, seed {seed}: step {k} "
                                              f"{step!r} diverged from the model: {e!r}; steps so far: {done!r}"}))
                sys.exit(0)
    print("RESULT " + json.dumps({"ok": True, "run_seq": drv.m.run_seq, "steps": len(steps)}))
    """
) % (ROOT, ROOT + "/tests")


def mirror(self, step, who):
    """The model's side of a step process `who` executes: its state changes, not its checks."""
    m = self.m
    kind = step[0]
    if kind == "corrupt":
        m.corrupt_word(step[1], step[2], step[3])
    elif kind == "landing":
        m.arm(step[1], step[2], step[3])
    elif kind == "opt" and step[1] in FAULTS:
        m.arm_measure(getattr(m, FAULTS[step[1]]), who, step[2])


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
