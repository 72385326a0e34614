"""Exact model of what one long-lived probe handle must report, for the sequence tests (no GPU).

A daemon keeps one handle for days and interleaves runs, option changes, remaps, fault injection and the on-demand
measurements on it.  `HandleModel` follows the same calls and says, from the pattern spec alone, what each one must
return: the expected values come from the CPU oracle (oracle/oracle.py), tests/word_ref.py, tests/latency_ref.py and
tests/bwcurve_ref.py, never from the library.  It tracks:

- the counters: run_seq and the call_seq of pingpong, atomics and bwcurve (a refused call advances none);
- the options in force: path, CTAs per rank, verify CTAs, the schedule flags, warm-up mode;
- the phase table each rank must walk (cdprobe_schedule with the current options, with the jobs of an unmapped pair
  idled as the library's schedule does);
- source corruptions at rest, {(rank, word): mask};
- every landing slot: the run that last wrote it (None: the zeros of open) and the landing-fault words xored in then;
- the unmapped (issuer, owner) pairs: a pair with either direction down has no read, write or warm-up job and no
  verify of its slots, so both cells read 0 (test_gpu_parity.py::test_unmapped_peer_gives_zero_cell_and_run_returns);
  only the unmapped direction carries CDPROBE_ERR_STATE in `status`, and the one-sided measurements (latency, atomics,
  bwcurve) skip only that direction.

The read checksum of a slice with corrupted words is the oracle's with, per corrupted word w (mask m, granule g from
the slice's start), S += (w ^ m) - w and X ^= rotl64(m, fold6(g)): X is a xor of rotated granule xors, and rotation
distributes over xor.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
from typing import Dict, List, Optional, Tuple

import numpy as np

import bwcurve_ref
import latency_ref
import word_ref

M64 = (1 << 64) - 1
SEED = 0xCD5EED0000000001
OP_READ, OP_WRITE = 1, 2
ERR_STATE = -9
ERR_INTEGRITY = -10
FLAG_OVERLAP_VERIFY = 0x20
FLAG_UNIDIRECTIONAL = 0x80
FLAG_SERIAL_VERIFY = 0x100
FLAG_ALL_RANK_BARRIERS = 0x400
FLAG_PAIR_BARRIERS = 0x800
KIND_NAMES = {0: "-", 1: "read", 2: "write", 3: "verify", 4: "warm"}
JOB_NONE, JOB_READ, JOB_WRITE, JOB_VERIFY, JOB_WARM = 0, 1, 2, 3, 4
# The checksum pass at open is the handle's first launch and takes sequence number 1, so the first run is 2.
FIRST_RUN_SEQ = 2


def rotl64(x: int, r: int) -> int:
    r %= 64
    return ((x << r) | (x >> (64 - r))) & M64 if r else x


def src_word(seed: int, rank: int, k: int) -> int:
    return int(word_ref.src_words(seed, rank, k, 1)[0])


def corrupted_checksum(base: Tuple[int, int], seed: int, rank: int, first: int, words: int,
                       corruptions: Dict[int, int]) -> Tuple[int, int]:
    """(S, X) of words [first, first + words) of rank's source buffer, given the clean (S, X) `base` and the masks
    xored into some words of that buffer ({word index: mask})."""
    s, x = base
    for k, m in corruptions.items():
        if first <= k < first + words:
            w = src_word(seed, rank, k)
            s = (s + ((w ^ m) - w)) & M64
            x ^= rotl64(m, word_ref.fold6((k - first) // word_ref.GRANULE_WORDS))
    return s, x


@dataclasses.dataclass
class Slot:
    run_seq: Optional[int] = None              # the run that last wrote the slot; None: never (zeros of open)
    faults: Tuple[Tuple[int, int], ...] = ()   # landing-fault (word, mask) xored in at that run


class HandleModel:
    """What one handle over `n` ranks must report.  `local` lists the global ranks this process drives (all of them
    in one process).  `oracle` is oracle/oracle.py; `schedule(n, rank, bytes, mode, ops, flags, ctas, verify_ctas)`
    returns an abi.ScheduleT (cdprobe_schedule)."""

    def __init__(self, oracle, schedule, n: int, nbytes: int, sm_count: int, ctas: int = 0, local=None,
                 flags: int = 0, seed: int = SEED, mode: int = 1, ops: int = 3):
        self.oracle, self._schedule = oracle, schedule
        self.n, self.nbytes, self.mode, self.ops, self.seed = n, nbytes, mode, ops, seed
        self.local = list(range(n)) if local is None else list(local)
        pl = oracle.plan(n, nbytes, mode, n == 1)
        self.bpp = pl.bytes_per_pair
        self.W = self.bpp // 8
        self.n_slices = pl.n_slices
        self.src_words = pl.src_bytes // 8
        self.rounds = pl.rounds
        self.diag = n == 1
        self.sm_count = sm_count
        self.flags = flags | FLAG_OVERLAP_VERIFY   # the overlapped verify is on unless SERIAL_VERIFY is asked for
        self.ctas = {g: ctas or sm_count for g in self.local}
        self.verify_ctas = 32
        self.path = 1 if flags & 0x08 else 0
        self.warm_mode = 1
        self.runs = 0                              # cdprobe_run calls that returned
        self.run_seq = 0                           # of the last run; 0: none yet
        self.pp_calls = self.at_calls = self.bw_calls = 0
        self.corrupt: Dict[Tuple[int, int], int] = {}      # (rank, word) -> mask, at rest
        # armed landing fault of each process's handle (one per handle): {process: (issuer, target, faults)}
        self.fault: Dict[int, Tuple[int, int, Tuple[Tuple[int, int], ...]]] = {}
        self.slots: Dict[Tuple[int, int], Slot] = {}
        self.unmapped = set()                      # (issuer, owner): issuer's mapping of owner torn down
        self._cache: Dict[Tuple[int, int, int], Tuple[int, int]] = {}

    # ---- geometry ------------------------------------------------------------------------------------------
    def slot_of(self, i: int, j: int) -> int:
        return self.n - 1 if i == j else (i if i < j else i - 1)

    def first_word(self, i: int, j: int) -> int:
        """Index of read cell (i, j)'s word 0 in j's source buffer."""
        return 0 if self.mode == 2 else self.slot_of(i, j) * self.W

    def cells(self) -> List[Tuple[int, int]]:
        return [(i, j) for i in range(self.n) for j in range(self.n) if i != j or self.diag]

    def pair_ok(self, i: int, j: int) -> bool:
        return (i, j) not in self.unmapped and (j, i) not in self.unmapped

    def maps(self, reader: int, target: int) -> bool:
        return reader == target or (reader, target) not in self.unmapped

    def status(self, i: int, j: int) -> int:
        return ERR_STATE if (i, j) in self.unmapped else 0

    # ---- expected values -----------------------------------------------------------------------------------
    def clean_checksum(self, rank: int, first: int, words: int) -> Tuple[int, int]:
        key = (rank, first, words)
        if key not in self._cache:
            self._cache[key] = self.oracle.src_checksum(self.seed, rank, first, words)
        return self._cache[key]

    def corruptions_of(self, rank: int) -> Dict[int, int]:
        return {k: m for (r, k), m in self.corrupt.items() if r == rank}

    def read_checksum(self, i: int, j: int, words: Optional[int] = None) -> Tuple[int, int]:
        """(S, X) of the first `words` (default: all) of read cell (i, j)'s region as it is at rest."""
        first, words = self.first_word(i, j), self.W if words is None else words
        return corrupted_checksum(self.clean_checksum(j, first, words), self.seed, j, first, words,
                                  self.corruptions_of(j))

    def read_clean(self, i: int, j: int, words: Optional[int] = None) -> bool:
        first, words = self.first_word(i, j), self.W if words is None else words
        return not any(first <= k < first + words for k in self.corruptions_of(j))

    def write_checksum(self, i: int, j: int, run_seq: int) -> Tuple[int, int]:
        return self.oracle.write_checksum(self.seed, i, j, run_seq, self.W)

    def phase_table(self, g: int) -> List[dict]:
        """The phases rank g's kernel walks: job kinds and peers (trace names), with an unmapped pair's jobs idled."""
        # cdprobe_schedule turns the overlapped verify on unless it is asked for the serial one
        flags = self.flags if self.flags & FLAG_OVERLAP_VERIFY else self.flags | FLAG_SERIAL_VERIFY
        s = self._schedule(self.n, g, self.nbytes, self.mode, self.ops, flags, self.ctas_of(g), self.verify_ctas)
        out = []
        for p in range(s.n_phases):
            ph = {}
            for jb in (0, 1):
                kind, peer = s.kind[jb][p], s.peer[jb][p]
                if kind in (JOB_READ, JOB_WRITE, JOB_WARM) and peer != g and not self.pair_ok(g, peer):
                    kind, peer = JOB_NONE, g
                if kind == JOB_VERIFY and s.writer[jb][p] != g and not self.pair_ok(g, s.writer[jb][p]):
                    kind = JOB_NONE
                ph["job%d" % jb], ph["peer%d" % jb] = KIND_NAMES[kind], peer
            out.append(ph)
        return out

    def ctas_of(self, g: int) -> int:
        return self.ctas.get(g, self.ctas[self.local[0]])

    # ---- calls ---------------------------------------------------------------------------------------------
    def run(self) -> dict:
        """Advance the handle by one cdprobe_run and return what every cell of the domain must hold:
        {"run_seq", "warmed" (None: depends on wall-clock idle time), "cells": {(i, j): {...}}}."""
        seq = FIRST_RUN_SEQ + self.runs
        first_run = self.runs == 0
        self.runs += 1
        self.run_seq = seq
        warmed = {0: False, 2: self.rounds > 0}.get(self.warm_mode, self.rounds > 0 if first_run else None)
        cells = {}
        for i in range(self.n):
            for j in range(self.n):
                if i == j and not self.diag:
                    cells[(i, j)] = dict(reach_read=1, reach_write=1, read=(0, 0), write=(0, 0), status=0, probed=False)
                    continue
                ok = self.pair_ok(i, j)
                c = dict(status=self.status(i, j), probed=ok)
                if ok:
                    c["read"] = self.read_checksum(i, j)
                    c["reach_read"] = int(self.read_clean(i, j))
                    c["write"] = self.write_checksum(i, j, seq)
                    f = self.fault.get(self.process_of(i))
                    armed = f is not None and f[:2] == (i, j)
                    c["reach_write"] = 0 if armed else 1
                    self.slots[(i, j)] = Slot(seq, f[2] if armed else ())
                else:
                    c.update(read=(0, 0), write=(0, 0), reach_read=0, reach_write=0)
                cells[(i, j)] = c
        return {"run_seq": seq, "warmed": warmed, "cells": cells}

    def diagnose(self, op: str, i: int, j: int):
        """(word_ref.Spec, observed words) of cell (op, i, j) after the last run."""
        assert self.run_seq, "no run yet"
        if op == "read":
            first = self.first_word(i, j)
            spec = word_ref.read_spec(self.seed, self.n, j, first, self.W, self.src_words)
            obs = word_ref.src_words(self.seed, j, first, self.W)
            for k, m in self.corruptions_of(j).items():
                if first <= k < first + self.W:
                    obs[k - first] ^= np.uint64(m)
            return spec, obs
        spec = word_ref.write_spec(self.seed, self.n, i, j, self.run_seq, self.W)
        return spec, self.slot_words(i, j)

    def slot_words(self, i: int, j: int) -> np.ndarray:
        """What landing slot (i, j) holds: the pattern of the run that last wrote it with that run's landing faults
        xored in, or zeros."""
        slot = self.slots.get((i, j), Slot())
        if slot.run_seq is None:
            return np.zeros(self.W, dtype=np.uint64)
        obs = word_ref.write_words(word_ref.write_salt(self.seed, i, j, slot.run_seq), 0, self.W)
        for k, m in slot.faults:
            obs[k] ^= np.uint64(m)
        return obs

    def latency(self, hops: int, reps: int) -> Dict[Tuple[int, int], dict]:
        """Per local-row cell: measured, status and (when measured) the digest of the chase over the words at rest."""
        lines = self.bpp // latency_ref.LINE_BYTES
        out = {}
        for i, j in self.cells():
            if i not in self.local:
                continue
            if not self.maps(i, j):
                out[(i, j)] = dict(measured=False, status=ERR_STATE)
                continue
            first = self.first_word(i, j)
            words = {k: src_word(self.seed, j, k) ^ m for k, m in self.corruptions_of(j).items()}
            d = latency_ref.digest(self.seed, i, j, first, lines, hops, reps, words)
            clean = d if not words else latency_ref.digest(self.seed, i, j, first, lines, hops, reps)
            out[(i, j)] = dict(measured=True, digest=d, status=0 if d == clean else ERR_INTEGRITY)
        return out

    def pingpong(self) -> Tuple[int, Dict[Tuple[int, int], dict]]:
        self.pp_calls += 1
        out = {}
        for i in self.local:
            for j in range(self.n):
                if i != j:
                    ok = self.pair_ok(i, j)
                    out[(i, j)] = dict(measured=ok, status=0 if ok else ERR_STATE)
        return self.pp_calls, out

    def atomics(self) -> Tuple[int, Dict[Tuple[int, int], dict]]:
        self.at_calls += 1
        out = {(i, j): dict(measured=self.maps(i, j), status=self.status(i, j))
               for i, j in self.cells() if i in self.local}
        return self.at_calls, out

    def bwcurve(self) -> Tuple[int, List[int], Dict[Tuple[int, int], dict]]:
        """call_seq, the size ladder, and per local-row cell: measured, status, bad_sizes and the (S, X) per size."""
        self.bw_calls += 1
        sizes = bwcurve_ref.ladder(self.bpp)
        out = {}
        for i, j in self.cells():
            if i not in self.local:
                continue
            if not self.maps(i, j):
                out[(i, j)] = dict(measured=False, status=ERR_STATE)
                continue
            bad = sum(1 << k for k, s in enumerate(sizes) if not self.read_clean(i, j, s // 8))
            out[(i, j)] = dict(measured=True, status=ERR_INTEGRITY if bad else 0, bad_sizes=bad,
                               sx=[self.read_checksum(i, j, s // 8) for s in sizes])
        return self.bw_calls, sizes, out

    # ---- state changes -------------------------------------------------------------------------------------
    def corrupt_word(self, rank: int, word: int, mask: int) -> None:
        m = self.corrupt.pop((rank, word), 0) ^ mask
        if m:
            self.corrupt[(rank, word)] = m

    def process_of(self, g: int) -> int:
        return g // len(self.local)

    def arm(self, i: int, j: int, faults) -> None:
        """cdprobe_corrupt_landing from issuer i: replaces the arming of i's handle; no faults disarms it."""
        if faults:
            self.fault[self.process_of(i)] = (i, j, tuple(sorted(faults)))
        else:
            self.fault.pop(self.process_of(i), None)

    def set_flag(self, flag: int, on: bool) -> None:
        self.flags = (self.flags & ~flag) | (flag if on else 0)

    def set_ctas(self, value: int) -> None:
        for g in self.local:
            self.ctas[g] = value or self.sm_count


def schedule_fn(lib, abi):
    """cdprobe_schedule as a function of its arguments, for HandleModel."""
    def schedule(n, rank, nbytes, mode, ops, flags, ctas, verify_ctas):
        s = abi.ScheduleT()
        rc = lib.cdprobe_schedule(n, rank, nbytes, mode, ops, flags, ctas, verify_ctas, C.byref(s))
        assert rc == 0, (n, rank, flags, ctas, verify_ctas, rc)
        return s
    return schedule
