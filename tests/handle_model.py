"""Exact model of what one long-lived probe handle must report, for the sequence tests (no GPU).

A daemon keeps one handle for days and interleaves runs, option changes, remaps, fault injection and the on-demand
measurements on it.  `HandleModel` follows the same calls and says, from the pattern spec alone, what each one must
return: the expected values come from the CPU oracle (oracle/oracle.py), tests/word_ref.py, tests/latency_ref.py,
tests/bwcurve_ref.py, tests/allreduce_ref.py, the all-reduce protocol references (allreduce_twoshot_ref,
allreduce_ll_ref, allreduce_ring_ref, allreduce_push_ref), tests/alltoall_ref.py, tests/memcpy_ref.py and
tests/ce_alltoall_ref.py, never from the library.  It tracks:

- the counters: run_seq and the call_seq of pingpong, atomics, bwcurve, the six all-reduces (one-shot, two-shot, LL,
  ring, push, NVLS), alltoall, memcpy and the copy-engine all-to-all (a refused call advances none); the NVLS call as
  it behaves where ranks share a device or a single rank's object is refused, so it runs nothing;
- each process's hardware queues per device, against which the copy-engine all-to-all is refused;
- the armed fault of each of those ladder measurements in each process's handle; which pairs were unmapped when the
  exchange area (shared by the all-to-all, memcpy and the copy-engine all-to-all, built by whichever is called first)
  was built, and the same for the two-shot's gather area and the LL, ring and push areas;
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
import os
import re
from typing import Dict, List, Optional, Tuple

import numpy as np

import allreduce_ll_ref
import allreduce_push_ref
import allreduce_ref
import allreduce_ring_ref
import allreduce_twoshot_ref
import alltoall_ref
import bwcurve_ref
import ce_alltoall_ref
import latency_ref
import memcpy_ref
import word_ref

M64 = (1 << 64) - 1
SEED = 0xCD5EED0000000001
OP_READ, OP_WRITE = 1, 2
ERR_ARG = -2
ERR_UNSUPPORTED = -8
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
CE_A2A_DEFAULT_REPS = 8


def max_connections(env) -> int:
    """The hardware queues per device cdprobe_open reads from CUDA_DEVICE_MAX_CONNECTIONS in `env`: its leading
    integer clamped to at most 32 when positive, else the CUDA runtime's default of 8."""
    m = re.match(r"\s*([+-]?\d+)", env.get("CUDA_DEVICE_MAX_CONNECTIONS") or "")
    v = int(m.group(1)) if m else 0
    return min(v, 32) if v > 0 else ce_alltoall_ref.DEFAULT_QUEUES


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


def refold(base: Tuple[int, int], changed: Dict[int, Tuple[int, int]], n_words: int) -> Tuple[int, int]:
    """(S, X) of the first n_words of a word array whose clean (S, X) is `base`, given the words that differ from the
    clean ones ({word: (old, new)}): S += new - old and X ^= rotl64(old ^ new, fold6(word's granule))."""
    s, x = base
    for k, (old, new) in changed.items():
        if k < n_words:
            s = (s + new - old) & M64
            x ^= rotl64(old ^ new, word_ref.fold6(k // word_ref.GRANULE_WORDS))
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
                 flags: int = 0, seed: int = SEED, mode: int = 1, ops: int = 3, timeout_ms: int = 20000):
        self.oracle, self._schedule = oracle, schedule
        self.timeout_ms = timeout_ms
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
        self.pp_calls = self.at_calls = self.bw_calls = self.a2a_calls = self.mc_calls = 0
        # the all-reduces' calls: one-shot, two-shot, LL, ring, push
        self.ar_calls = self.ts_calls = self.ll_calls = self.ring_calls = self.push_calls = 0
        # the armed fault option of each measurement in each process's handle, {process: value} (absent: disarmed):
        # CDPROBE_OPT_ALLREDUCE_FAULT, _ALLREDUCE_{TWOSHOT,LL,RING,PUSH}_FAULT, _ALLTOALL_FAULT, _MEMCPY_FAULT
        self.ar_fault: Dict[int, int] = {}
        self.ts_fault: Dict[int, int] = {}
        self.ll_fault: Dict[int, int] = {}
        self.ring_fault: Dict[int, int] = {}
        self.push_fault: Dict[int, int] = {}
        self.a2a_fault: Dict[int, int] = {}
        self.mc_fault: Dict[int, int] = {}
        # the copy-engine all-to-all: its calls, its armed fault (CDPROBE_OPT_CE_ALLTOALL_FAULT) per process, each
        # process's hardware queues per device (CUDA_DEVICE_MAX_CONNECTIONS as read by cdprobe_open; by default this
        # process's, for every process) and each global rank's device ordinal (absent: 0), which the caller sets from
        # the ordinals the handle was opened with
        self.cea_calls = 0
        self.cea_fault: Dict[int, int] = {}
        # the NVLS all-reduce: its calls, its armed fault (CDPROBE_OPT_ALLREDUCE_NVLS_FAULT) per process, and whether
        # the driver refuses a multicast object of one device (the caller sets it from a one-rank call where it matters)
        self.nvls_calls = 0
        self.nvls_fault: Dict[int, int] = {}
        self.one_device_nvls_refused = True
        limit = max_connections(os.environ)
        self.max_connections: Dict[int, int] = {p: limit for p in range(n // len(self.local))}
        self.ordinal: Dict[int, int] = {}
        # the pairs unmapped when the first all-to-all, memcpy or copy-engine all-to-all built the exchange area they
        # share (None: not built yet); the area is mapped only where the probe mapping was up then, and remaps do not
        # map it later
        self.area_down: Optional[frozenset] = None
        # the same for the gather, LL, ring and push areas, each built by its own all-reduce's first call
        self.ar_area_down: Dict[str, Optional[frozenset]] = {"ts": None, "ll": None, "ring": None, "push": None}
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

    def ar_word(self, w: int) -> int:
        """Word w of the clean all-reduce output: the sum of word w of every rank's pattern."""
        return sum(src_word(self.seed, j, w) for j in range(self.n)) & M64

    def src_at_rest(self, rank: int, lo: int, hi: int) -> np.ndarray:
        """Words [lo, hi) of rank's source buffer as they are at rest."""
        w = word_ref.src_words(self.seed, rank, lo, hi - lo)
        for k, m in self.corruptions_of(rank).items():
            if lo <= k < hi:
                w[k - lo] ^= np.uint64(m)
        return w

    def _ar_set(self, words: Dict[int, Tuple[int, int]], lo: int, hi: int, fn) -> None:
        """Words [lo, hi) of one rep's all-reduce output {word: (clean, value)} (a word absent holds its clean sum)
        become fn(word, value) mod 2^64."""
        clean = sum(word_ref.src_words(self.seed, j, lo, hi - lo) for j in range(self.n))
        for i, w in enumerate(range(lo, hi)):
            c, v = words.get(w, (int(clean[i]),) * 2)
            words[w] = (c, fn(w, v) & M64)

    def _allreduce(self, name: str, reps: int, sizes: List[int], decode, effect, every_rep: bool = True):
        """One call of an all-reduce, on the rules they share.  name: the prefix of its armed faults ({process: value},
        `<name>_fault`) and its counter (`<name>_calls`); it has a shared area when ar_area_down has the name.
        decode(value, sizes) is the call's verdict on an armed value: None refuses it (CDPROBE_ERR_ARG, nothing
        advances), else a tuple whose first field is the rank in whose process it acts and whose second is its size.
        effect(words, unstored, row, size, fault) applies the fault to that row's output of timed rep 1 of the size
        ({word: (clean, value)}), or names output words the row never stores in the size (`unstored`).

        The area is built by the first call that is not refused, mapped only where the probe mapping was up then.  Any
        unmapped pair, or a pair down when the area was built, stops every rank, and call_seq still advances.  Otherwise
        output word w is the sum of word w of every source buffer as it is at rest (slice 0 only), and a word is bad
        when it differs from the clean sum.  every_rep: every rep, warm-up included, is checked and cleared, so
        bad_words and first_bad cover every rep; else (the LL) only the last rep of a size is.  The reported (S, X) is
        the last timed rep's, so it shows a fault of timed rep 1 when reps is 1, and a size fails when any rep's (S, X)
        or any checked word is wrong."""
        faults = []
        for proc, v in getattr(self, name + "_fault").items():
            f = decode(v, sizes)
            if f is None:
                return None
            if self.process_of(f[0]) == proc:
                faults.append(f)
        faults.sort(key=lambda f: f[-1])  # the push's all-gather fault (mode 3) acts after the contributions
        if name in self.ar_area_down and self.ar_area_down[name] is None:
            self.ar_area_down[name] = frozenset(self.unmapped)
        seq = getattr(self, name + "_calls") + 1
        setattr(self, name + "_calls", seq)
        out = dict(call_seq=seq, sizes=sizes, rows={})
        if self.unmapped or self.ar_area_down.get(name):
            for g in self.local:
                out["rows"][g] = dict(measured=False, status=ERR_STATE)
            return out
        clean = allreduce_ref.expected(self.seed, self.n, tuple(sizes))
        delta: Dict[int, int] = {}
        for (r, k), m in self.corrupt.items():
            if k < self.W:
                w = src_word(self.seed, r, k)
                delta[k] = (delta.get(k, 0) + (w ^ m) - w) & M64
        at_rest = {}  # {output word: (clean, as summed)} of the words the corruptions change
        for w, d in delta.items():
            if d:
                c = self.ar_word(w)
                at_rest[w] = (c, (c + d) & M64)
        for g in self.local:
            row = dict(measured=True, bad_sizes=0, sx=[], bad_words=[], first_bad=[])
            for k, s in enumerate(sizes):
                nw = s // 8
                rep1, unstored = dict(at_rest), set()
                for f in faults:
                    if f[1] == k:
                        effect(rep1, unstored, g, s, f)
                last = rep1 if reps == 1 else at_rest
                if every_rep:
                    bad = sorted(w for w, (o, v) in at_rest.items() if w < nw and o != v)
                    bad1 = sorted(w for w, (o, v) in rep1.items() if w < nw and o != v)
                    n_bad = reps * len(bad) + len(bad1)  # the warm-up and reps 2.. see the words at rest
                    first = min(bad[:1] + bad1[:1], default=None)
                else:
                    seen = dict(last)
                    for w in unstored:  # the output starts zeroed and every check clears it
                        seen[w] = (seen.get(w, (self.ar_word(w),))[0], 0)
                    bad = sorted(w for w, (o, v) in seen.items() if w < nw and o != v)
                    n_bad, first = len(bad), (bad[0] if bad else None)
                sx = refold(clean[k], last, nw)
                row["sx"].append(sx)
                row["bad_words"].append(n_bad)
                row["first_bad"].append(word_ref.U64_MAX if first is None else 8 * first)
                if n_bad or refold(clean[k], rep1, nw) != clean[k] or refold(clean[k], at_rest, nw) != clean[k]:
                    row["bad_sizes"] |= 1 << k
            row["status"] = ERR_INTEGRITY if row["bad_sizes"] else 0
            out["rows"][g] = row
        return out

    def allreduce(self, reps: int) -> Optional[dict]:
        """What cdprobe_allreduce with `reps` timed reps must return: {"call_seq", "sizes", "rows": {local rank: {...}}},
        or None when some process's armed fault names no rank, size or word of the ladder.  An armed fault acts in
        timed rep 1 of its size on its rank: it adds 1 to its word, or (drop, bit 48) leaves its 8 KiB unit unstored,
        which the check after the rep reads as 0s.  The rest is _allreduce's."""
        sizes = bwcurve_ref.ladder(self.bpp)

        def decode(v, sizes):
            fr, fk, fw = (v >> 32) & 0xFFFF, (v >> 24) & 0xFF, v & 0xFFFFFF
            if v >> 49 or fr == 0 or fr > self.n or fk == 0 or fk > len(sizes) or fw >= sizes[fk - 1] // 8:
                return None
            return fr - 1, fk - 1, fw, bool(v >> 48)

        def effect(words, unstored, g, s, f):
            rank, _, fw, drop = f
            if g != rank:
                return
            if drop:
                unit = allreduce_ref.unit_words(fw, s)
                self._ar_set(words, unit.start, unit.stop, lambda w, v: 0)
            else:
                self._ar_set(words, fw, fw + 1, lambda w, v: v + 1)

        return self._allreduce("ar", reps, sizes, decode, effect)

    def twoshot(self, reps: int) -> Optional[dict]:
        """cdprobe_allreduce_twoshot, as allreduce().  Its fault (receiver, size, word, drop) acts in the process that
        hosts the rank whose chunk holds the word: timed rep 1 delivers the word to the receiver xored with 1, or (drop)
        none of its 8 KiB unit, which the receiver's check reads as 0s.  It has a gather area."""
        sizes = bwcurve_ref.ladder(self.bpp)

        def decode(v, sizes):
            fr, fk, fw = (v >> 32) & 0xFFFF, (v >> 24) & 0xFF, v & 0xFFFFFF
            if v >> 49 or fr == 0 or fr > self.n or fk == 0 or fk > len(sizes) or fw >= sizes[fk - 1] // 8:
                return None
            return allreduce_twoshot_ref.owner(sizes[fk - 1], self.n, fw), fk - 1, fr - 1, fw, bool(v >> 48)

        def effect(words, unstored, g, s, f):
            _, _, recv, fw, drop = f
            if g != recv:
                return
            if drop:
                unit = allreduce_ref.unit_words(fw, s)
                self._ar_set(words, unit.start, unit.stop, lambda w, v: 0)
            else:
                self._ar_set(words, fw, fw + 1, lambda w, v: v ^ 1)

        return self._allreduce("ts", reps, sizes, decode, effect)

    def ll(self, reps: int) -> Optional[dict]:
        """cdprobe_allreduce_ll, on its own ladder (cut at 1 MiB).  Its fault (mode, sender, receiver, size, arg) acts
        in the process that hosts the sender: mode 0, in timed rep 1 the packet of word arg to the receiver carries the
        sender's salted input xored with 1, which moves the receiver's word by +1 or -1; mode 1, the sender waits arg us
        (no value changes); mode 2, the receiver (which is the sender) stores nothing to word arg in any rep of the size
        and still folds the word into (S, X).  Only the last rep of a size is word-checked.  It has an LL area."""
        sizes = allreduce_ll_ref.ladder(self.bpp)

        def decode(v, sizes):
            mode, fs, fr, fk, arg = v >> 48, (v >> 40) & 0xFF, (v >> 32) & 0xFF, (v >> 24) & 0xFF, v & 0xFFFFFF
            if (mode > 2 or fs == 0 or fs > self.n or fr == 0 or fr > self.n or fk == 0 or fk > len(sizes)
                    or (mode != 1 and arg >= sizes[fk - 1] // 8) or (mode == 0 and fs == fr) or (mode == 2 and fs != fr)
                    or (mode == 1 and 2 * arg >= 1000 * self.timeout_ms)):
                return None
            return fs - 1, fk - 1, fr - 1, arg, mode

        def effect(words, unstored, g, s, f):
            sender, k, recv, arg, mode = f
            if g != recv or mode == 1:
                return
            if mode == 2:
                unstored.add(arg)
                return
            fl = allreduce_ll_ref.flag(self.ll_calls, k, 1)
            v = (int(self.src_at_rest(sender, arg, arg + 1)[0]) + allreduce_ll_ref.salt(self.seed, sender, fl)) & M64
            self._ar_set(words, arg, arg + 1, lambda w, x: x + (v ^ 1) - v)

        return self._allreduce("ll", reps, sizes, decode, effect, every_rep=False)

    def ring(self, reps: int) -> Optional[dict]:
        """cdprobe_allreduce_ring.  Its fault (mode, phase, sender, size, arg) acts in the process that hosts the sender,
        in timed rep 1: mode 0, the sender's push of word arg carries it xored with 1; mode 1, that push stores nothing
        of the word's unit; mode 2, the sender waits arg us (no value changes).  The rows it fails and what they then
        hold are allreduce_ring_ref's: in the reduce-scatter the sender's partial of the chunk is off in every row; in
        the all-gather the rows downstream of the hop hold the word xored with 1, or in place of the unit what they got
        in the reduce-scatter (the sender's partial, or the clear's 0s).  It has a ring area."""
        sizes = bwcurve_ref.ladder(self.bpp)
        n = self.n

        def decode(v, sizes):
            mode, phase, fs, fk, arg = v >> 48, (v >> 40) & 0xFF, (v >> 32) & 0xFF, (v >> 24) & 0xFF, v & 0xFFFFFF
            if mode > 2 or phase > 1 or fs == 0 or fs > n or fk == 0 or fk > len(sizes):
                return None
            if mode == 2 and 2 * arg >= 1000 * self.timeout_ms:
                return None
            if mode < 2 and (n == 1 or arg >= sizes[fk - 1] // 8 or allreduce_ring_ref.chunk_of(sizes[fk - 1], n, arg)
                             not in allreduce_ring_ref.pushes(n, fs - 1, phase)):
                return None
            return fs - 1, fk - 1, arg, phase, mode

        def effect(words, unstored, g, s, f):
            sender, _, word, phase, mode = f
            if mode == 2 or g not in allreduce_ring_ref.failing_rows(n, sender, phase, s, word):
                return
            if phase == 1 and mode == 0:
                self._ar_set(words, word, word + 1, lambda w, v: v ^ 1)
                return
            unit = allreduce_ref.unit_words(word, s)
            c = allreduce_ring_ref.chunk_of(s, n, word)
            part = None  # the sender's partial of chunk c: the inputs of ranks sender - s' .. sender, as they are at rest
            if sender != c:
                part = sum(self.src_at_rest(j, unit.start, unit.stop)
                           for j in allreduce_ring_ref.partial_ranks(n, sender, c))
            p = {w: int(part[w - unit.start]) for w in unit} if part is not None else {w: 0 for w in unit}
            if phase == 1:
                self._ar_set(words, unit.start, unit.stop, lambda w, v: p[w])
            elif mode == 0:
                self._ar_set(words, word, word + 1, lambda w, v: v + (p[w] ^ 1) - p[w])
            else:
                self._ar_set(words, unit.start, unit.stop, lambda w, v: v - p[w])

        return self._allreduce("ring", reps, sizes, decode, effect)

    def push(self, reps: int) -> Optional[dict]:
        """cdprobe_allreduce_push.  Its fault (mode, rank, size, word) acts in timed rep 1 (allreduce_push_ref): modes
        0-2 in the process that hosts sender `rank`, which contributes its word + 1 (every row's word + 1), skips the
        word's unit (every row's unit less the sender's input) or reduces it twice (plus the input); mode 3 in the
        process that hosts the word's owner, which pushes the word xored with 1 to receiver `rank`.  It has a push
        area."""
        sizes = bwcurve_ref.ladder(self.bpp)
        n = self.n

        def decode(v, sizes):
            mode, fr, fk, fw = v >> 48, (v >> 32) & 0xFFFF, (v >> 24) & 0xFF, v & 0xFFFFFF
            if mode > 3 or fr == 0 or fr > n or fk == 0 or fk > len(sizes) or fw >= sizes[fk - 1] // 8:
                return None
            if mode < 3:
                return fr - 1, fk - 1, fr - 1, fw, mode
            owner = allreduce_push_ref.word_owner(sizes[fk - 1], n, fw)
            return None if n == 1 or owner == fr - 1 else (owner, fk - 1, fr - 1, fw, mode)

        def effect(words, unstored, g, s, f):
            _, _, rank, fw, mode = f
            if mode == 0:
                self._ar_set(words, fw, fw + 1, lambda w, v: v + 1)
            elif mode == 3:
                if g == rank:
                    self._ar_set(words, fw, fw + 1, lambda w, v: v ^ 1)
            else:
                unit = allreduce_ref.unit_words(fw, s)
                x = self.src_at_rest(rank, unit.start, unit.stop)
                sign = -1 if mode == 1 else 1
                self._ar_set(words, unit.start, unit.stop, lambda w, v: v + sign * int(x[w - unit.start]))

        return self._allreduce("push", reps, sizes, decode, effect)

    def nvls_modelled(self) -> bool:
        """Whether the domain cannot form a multicast object, which is all allreduce_nvls models: two ranks share a
        device (by ordinal; a team holds each device once), or one rank whose one-device object the driver refuses."""
        if self.n == 1:
            return self.one_device_nvls_refused
        ordinals = [self.ordinal.get(g, 0) for g in range(self.n)]
        return len(set(ordinals)) < len(ordinals)

    def allreduce_nvls(self, reps: int, proc: int = 0):
        """What cdprobe_allreduce_nvls with `reps` timed reps must return in process `proc`, on a domain that cannot
        form a multicast object: every rank on one device (a team holds each device once), or one rank, whose
        one-device object the driver refuses.  A refused call returns CDPROBE_ERR_ARG with the text cdprobe_last_error
        then holds, which this returns, and advances nothing.  The refusals come in this order: reps above 64, then this
        process's armed fault (a mode above 1, bits 32 to 47 set, no size of the ladder, no word of its size), then
        another process's.  Otherwise the call advances its own call_seq and every local row reports
        CDPROBE_ERR_UNSUPPORTED, unmeasured, whatever the mappings: no NVLS area is built and nothing else changes.
        A domain that can form the object (nvls_modelled false) runs the kernel, which this does not model."""
        assert self.nvls_modelled(), "the NVLS call runs on this domain; the model covers only domains that refuse it"
        sizes = bwcurve_ref.ladder(self.bpp)
        if reps > 64:
            return "reps must be at most 64"

        def refusal(v):
            fk, word = (v >> 24) & 0xFF, v & 0xFFFFFF
            if v >> 48 > 1:
                return "the armed NVLS all-reduce fault has a mode above 1"
            if (v >> 32) & 0xFFFF:
                return "the armed NVLS all-reduce fault sets bits 32 to 47, which name nothing"
            if fk == 0 or fk > len(sizes):
                return "the armed NVLS all-reduce fault names no size of this call"
            if word >= sizes[fk - 1] // 8:
                return "the armed NVLS all-reduce fault names no output word of its size"
            return None

        why = {p: refusal(v) for p, v in self.nvls_fault.items()}
        if why.get(proc):
            return why[proc]
        if any(why.values()):
            return "another process called cdprobe_allreduce_nvls with invalid arguments"
        self.nvls_calls += 1
        return dict(call_seq=self.nvls_calls, sizes=sizes,
                    rows={g: dict(measured=False, status=ERR_UNSUPPORTED) for g in self.local})

    def build_area(self) -> None:
        """The exchange area, built by the first all-to-all, memcpy or copy-engine all-to-all call that is not
        refused."""
        if self.area_down is None:
            self.area_down = frozenset(self.unmapped)

    def _block(self, op: int, g: int, j: int, sizes: List[int], reps: int, fault=None) -> dict:
        """What the checks of cell (issuer g, target j)'s block report when the block is copied and checked in every
        rep, as cdprobe_memcpy and cdprobe_ce_alltoall both do: {"bad_sizes", "sx", "bad_words", "first_bad",
        "status"}.  The block holds its source slice (memcpy_ref.cell) as it is at rest after every rep, warm-up
        included, and is checked and cleared then: a corrupted word is one bad word per rep.  `fault` (k, word, mode)
        acts in timed rep 1 of size k: mode 0 overwrites the landed word with its pattern value xored with 1, mode 1
        copies nothing, so the cleared block reads as 0s.  The (S, X) is the last timed rep's."""
        c = memcpy_ref.cell(self.n, self.bpp, self.mode, op, g, j)
        src, first = c["src_rank"], c["first_word"]
        corr = {k - first: m for k, m in self.corruptions_of(src).items() if first <= k < first + self.W}
        cell = dict(bad_sizes=0, sx=[], bad_words=[], first_bad=[])
        fk, fw, mode = fault if fault is not None else (None, None, None)
        for k, s in enumerate(sizes):
            nw = s // 8
            clean_sx = self.clean_checksum(src, first, nw)
            rest = {}  # {destination word: (pattern, landed)} of the corrupted words of the prefix
            for w, m in corr.items():
                if w < nw:
                    p = src_word(self.seed, src, first + w)
                    rest[w] = (p, p ^ m)
            bad = sorted(rest)
            if fk == k and mode == 1:  # nothing landed: every word the pattern does not make 0 is bad
                pattern = word_ref.src_words(self.seed, src, first, nw)
                bad1, sx1 = [int(w) for w in np.flatnonzero(pattern != 0)], (0, 0)
            else:
                rep1 = dict(rest)
                if fk == k:
                    p = src_word(self.seed, src, first + fw)
                    rep1[fw] = (p, p ^ 1)
                bad1, sx1 = sorted(rep1), refold(clean_sx, rep1, nw)
            sx_rest = refold(clean_sx, rest, nw)
            cell["sx"].append(sx1 if reps == 1 else sx_rest)
            cell["bad_words"].append(reps * len(bad) + len(bad1))
            first_bad = min(bad[:1] + bad1[:1], default=None)
            cell["first_bad"].append(word_ref.U64_MAX if first_bad is None else 8 * first_bad)
            if bad or bad1 or sx1 != clean_sx or sx_rest != clean_sx:
                cell["bad_sizes"] |= 1 << k
        cell["status"] = ERR_INTEGRITY if cell["bad_sizes"] else 0
        return cell

    def memcpy(self, op: int, reps: int) -> Optional[dict]:
        """What cdprobe_memcpy with op and `reps` timed reps must return, or None when the op is neither OP_READ nor
        OP_WRITE or some process's armed fault names no cell, size or word, or has a mode above 1 (CDPROBE_ERR_ARG;
        nothing advances, and the exchange area is not built).  {"call_seq", "sizes", "cells": {(issuer, target):
        {...}}} for every cell whose issuer is local.  A cell runs when its issuer maps the target now and mapped it
        when the exchange area was built (by this call, an all-to-all or an earlier memcpy); else it is not measured and
        carries CDPROBE_ERR_STATE.  The destination of a cell that runs holds its source slice (memcpy_ref.cell) as it
        is at rest after every rep, warm-up included, and is checked and cleared then: a corrupted word is one bad word
        per rep.  An armed fault acts in the process that hosts its issuer, in timed rep 1 of its cell and size: mode 0
        overwrites one landed word with its pattern value xored with 1, mode 1 copies nothing, so the cleared
        destination reads as 0s.  The (S, X) is the last timed rep's."""
        n = self.n
        sizes = bwcurve_ref.ladder(self.bpp)
        if op not in (OP_READ, OP_WRITE):
            return None
        faults = {}
        for proc, v in self.mc_fault.items():
            mode, fi, ft, fk, fw = v >> 48, (v >> 40) & 0xFF, (v >> 32) & 0xFF, (v >> 24) & 0xFF, v & 0xFFFFFF
            if (mode > 1 or fi == 0 or fi > n or ft == 0 or ft > n or (fi == ft and not self.diag) or fk == 0
                    or fk > len(sizes) or fw >= sizes[fk - 1] // 8):
                return None
            if self.process_of(fi - 1) == proc:
                faults[(fi - 1, ft - 1)] = (fk - 1, fw, mode)
        self.build_area()
        self.mc_calls += 1
        cells = {}
        for g in self.local:
            for j in range(n):
                if g == j and not self.diag:
                    continue
                if (g, j) in self.unmapped or (g, j) in (self.area_down or ()):
                    cells[(g, j)] = dict(measured=False, status=ERR_STATE)
                    continue
                cells[(g, j)] = dict(measured=True, **self._block(op, g, j, sizes, reps, faults.get((g, j))))
        return dict(call_seq=self.mc_calls, sizes=sizes, cells=cells)

    def a2a_runs(self, s: int, d: int) -> bool:
        """Whether all-to-all cell (sender s, receiver d) runs: it exists, s maps d now, and s's view of d's exchange
        area was mapped when the area was built."""
        return ((s != d or self.diag) and (s, d) not in self.unmapped and self.area_down is not None
                and (s, d) not in self.area_down)

    def alltoall(self, reps: int) -> Optional[dict]:
        """What cdprobe_alltoall with `reps` timed reps must return, or None when some process's armed fault names no
        cell, size or word (CDPROBE_ERR_ARG; nothing advances, and the exchange area is not built).  {"call_seq",
        "sizes", "ranks": {local rank: {"measured", "blocks"}}, "cells": {(s, d): {...}}} with every cell whose receiver
        is local, and every cell that does not run whose sender is local.  The area is built by the first call that
        runs, so a pair unmapped then stays skipped after its remap.  Source corruptions and landing faults do not
        touch the blocks; an armed fault fails exactly its cell and size (the word check of every rep sees rep 1; the
        (S, X) of the last rep sees it when reps is 1)."""
        n = self.n
        sizes = bwcurve_ref.ladder(self.bpp)
        faults = {}
        for proc, v in self.a2a_fault.items():
            fs, fr, fk, fw = v >> 40, (v >> 32) & 0xFF, (v >> 24) & 0xFF, v & 0xFFFFFF
            if (fs == 0 or fs > n or fr == 0 or fr > n or (fs == fr and not self.diag) or fk == 0 or fk > len(sizes)
                    or fw >= sizes[fk - 1] // 8):
                return None
            if self.process_of(fs - 1) == proc:
                faults[(fs - 1, fr - 1)] = (fk - 1, fw)
        self.build_area()
        self.a2a_calls += 1
        seq = self.a2a_calls
        runs = self.a2a_runs
        ranks = {}
        for g in self.local:
            joined = any(runs(g, j) or runs(j, g) for j in range(n))
            ranks[g] = dict(measured=joined, blocks=sum(runs(g, j) for j in range(n)))
        cells = {}
        for s in range(n):
            for d in range(n):
                if (s == d and not self.diag) or not (d in self.local or (s in self.local and not runs(s, d))):
                    continue
                if not runs(s, d):
                    cells[(s, d)] = dict(cell_measured=False, cell_status=ERR_STATE)
                    continue
                sx = alltoall_ref.expected(self.seed, s, d, seq, reps, sizes)
                bad_words, first_bad = [0] * len(sizes), [word_ref.U64_MAX] * len(sizes)
                if (s, d) in faults:
                    fk, fw = faults[(s, d)]
                    bad_words[fk], first_bad[fk] = 1, 8 * fw
                    if reps == 1:
                        salt = word_ref.write_salt(self.seed, s, d, alltoall_ref.alltoall_seq(seq, fk, 1))
                        w = int(word_ref.write_words(salt, fw, 1)[0])
                        sx[fk] = refold(sx[fk], {fw: (w, w ^ 1)}, sizes[fk] // 8)
                bad = sum(1 << k for k, b in enumerate(bad_words) if b)
                cells[(s, d)] = dict(cell_measured=True, cell_status=ERR_INTEGRITY if bad else 0, bad_sizes=bad,
                                     bad_words=bad_words, first_bad=first_bad, sx=sx)
        return dict(call_seq=seq, sizes=sizes, ranks=ranks, cells=cells)

    def ce_alltoall(self, op: int, reps: int):
        """What cdprobe_ce_alltoall with op and `reps` timed reps (0: 8) must return, but the times.  A refused call
        returns its error code and advances nothing, nor builds the exchange area: ERR_ARG when reps is above 64, else
        when the op is neither OP_READ nor OP_WRITE, else when some process's armed fault names no cell, size or word
        (modes 0 and 1) or delay (mode 2, below timeout_ms / 2), or has a mode above 2; ERR_UNSUPPORTED when some
        process would hold more streams on one device than its CUDA_DEVICE_MAX_CONNECTIONS gives (ce_alltoall_ref.queues
        against max_connections).  Otherwise the call builds the area and advances call_seq.  When any probe mapping is
        down, or was down when the area was built, nothing runs: every local rank, and every cell with a local issuer or
        target, carries CDPROBE_ERR_STATE.  Else every rank issues every cell, and per cell whose owner (the issuer on a
        pull, the target on a push) is local the block's checks are memcpy's (_block) with the fault, of modes 0 and 1,
        armed in the process that hosts the issuer; mode 2 only delays a copy.
        {"call_seq", "sizes", "area_min_bytes" (n blocks; the area is that rounded up to the VMM granule the driver
        reports), "ranks": {local rank: {"measured", "status", "blocks"}}, "cells":
        {(issuer, target): {"cell_measured", "cell_status", ...}}}."""
        n = self.n
        sizes = bwcurve_ref.ladder(self.bpp)
        if reps > 64 or op not in (OP_READ, OP_WRITE):
            return ERR_ARG
        reps = reps or CE_A2A_DEFAULT_REPS
        faults = {}
        for proc, v in self.cea_fault.items():
            mode, fi, ft, fk, arg = v >> 48, (v >> 40) & 0xFF, (v >> 32) & 0xFF, (v >> 24) & 0xFF, v & 0xFFFFFF
            if (mode > 2 or fi == 0 or fi > n or ft == 0 or ft > n or (fi == ft and not self.diag) or fk == 0
                    or fk > len(sizes) or (mode < 2 and arg >= sizes[fk - 1] // 8)
                    or (mode == 2 and 2 * arg >= 1000 * self.timeout_ms)):
                return ERR_ARG
            if self.process_of(fi - 1) == proc and mode < 2:
                faults[(fi - 1, ft - 1)] = (fk - 1, arg, mode)
        n_procs = n // len(self.local)
        for proc in range(n_procs):
            ranks = range(proc * len(self.local), (proc + 1) * len(self.local))
            need, _ = ce_alltoall_ref.queues(n, self.diag, [self.ordinal.get(g, 0) for g in ranks])
            if need > self.max_connections[proc]:
                return ERR_UNSUPPORTED
        self.build_area()
        self.cea_calls += 1
        out = dict(call_seq=self.cea_calls, sizes=sizes, area_min_bytes=n * self.bpp, ranks={}, cells={})
        if self.unmapped or self.area_down:
            for g in self.local:
                out["ranks"][g] = dict(measured=False, status=ERR_STATE, blocks=0)
                for j in range(n):
                    if j != g or self.diag:
                        out["cells"][(g, j)] = out["cells"][(j, g)] = dict(cell_measured=False, cell_status=ERR_STATE)
            return out
        for g in self.local:
            out["ranks"][g] = dict(measured=True, status=0, blocks=n - 1 + self.diag)
        for g, j in ce_alltoall_ref.cells(n, self.diag):
            if ce_alltoall_ref.owner(op, g, j) in self.local:
                b = self._block(op, g, j, sizes, reps, faults.get((g, j)))
                out["cells"][(g, j)] = dict(cell_measured=True, cell_status=b.pop("status"), **b)
        return out

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

    def arm_measure(self, faults: Dict[int, int], proc: int, value: int) -> None:
        """CDPROBE_OPT_ALLREDUCE_FAULT or CDPROBE_OPT_ALLTOALL_FAULT (`faults` is ar_fault or a2a_fault) set to `value`
        in process proc's handle; 0 disarms it.  The value is only checked by the next call."""
        if value:
            faults[proc] = value
        else:
            faults.pop(proc, None)

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
