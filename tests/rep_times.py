"""The rep-record fold of measure.cc, run on the host: summarize, ladder_times, bw_times and bw_summarize turn the rep
records a kernel (or the events of a copy) left into the times, summary and verdict every ladder measurement, latency,
pingpong and atomics report.

generate() copies the four templates out of csrc/measure.cc verbatim; each must be found exactly once, so an edit to
any of them reaches the copy or fails loudly.  build() compiles the copy with tests/c/rep_times_host.cc against the
real cdprobe.h, bwcurve.h, timed_rep.cuh and probe_types.h into one shared library, and Fold drives it with records the
test builds by hand.  The restatements at the end say in plain Python what each function must give.

MUTATIONS are deliberate one-line errors in the copy, for checking that test_rep_times_cpu.py sees each:
  bw_times_previous_rel   a rep's window opens at the previous rep's release (t_rel[k][r - 1])
  warmup_in_stats         summarize and bw_times sort the warm-up rep (r = 0) into the times and drop the last rep
  median_low              ladder_times takes its median at (reps - 1) / 2"""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "k8s-dra-driver-gpu_b200", "csrc")
MEASURE = os.path.join(CSRC, "measure.cc")
HOST = os.path.join(HERE, "c", "rep_times_host.cc")
CUDA_INCLUDE = "/usr/local/cuda/include"  # cuda_runtime.h, which bwcurve.h includes for its launcher declarations
FUNCTIONS = ("summarize", "ladder_times", "bw_times", "bw_summarize")

ERR_TIMEOUT, ERR_INTEGRITY = -5, -10  # CDPROBE_ERR_TIMEOUT, CDPROBE_ERR_INTEGRITY (pinned in test_rep_times_cpu.py)

# name: [(function, text in it, its replacement)]; each text occurs in its function
MUTATIONS = {
    "bw_times_previous_rel": [("bw_times", "s.t_rel[k][r])", "s.t_rel[k][r - 1])")],
    "warmup_in_stats": [("summarize", "if (k > 0) ns[k - 1] = ", "if (k < reps) ns[k] = "),
                        ("bw_times", "for (uint32_t r = 1; r <= reps; ++r) ns[k][r - 1] =",
                         "for (uint32_t r = 0; r < reps; ++r) ns[k][r] =")],
    "median_low": [("ladder_times", "[reps / 2]", "[(reps - 1) / 2]")],
}


def extract(text=None):
    """{name: source} of the four templates in measure.cc, each from its `template <typename Out>` line to its closing
    brace at column 0.  Asserts that each is found exactly once."""
    if text is None:
        with open(MEASURE) as f:
            text = f.read()
    out = {}
    for name in FUNCTIONS:
        found = re.findall(r"^template <typename Out>\nstatic \w+ " + name + r"\(.*?^\}\n", text, re.S | re.M)
        assert len(found) == 1, f"{name}: found {len(found)} times in measure.cc"
        out[name] = found[0]
    return out


def generate(mutation=None):
    """The four templates, in measure.cc's order, with `mutation` applied (every occurrence of each of its texts in
    its function)."""
    funcs = extract()
    for name, old, new in MUTATIONS[mutation] if mutation is not None else ():
        assert old in funcs[name], (mutation, name, old)
        funcs[name] = funcs[name].replace(old, new)
    return "\n".join(funcs[name] for name in FUNCTIONS)


def build(out_dir, mutation=None):
    """Compiles the copy with the host harness into out_dir/librep_times.so and returns its path.  Skips the calling
    test when g++ or the CUDA headers are missing."""
    import pytest

    gxx = shutil.which("g++")
    if gxx is None or not os.path.exists(os.path.join(CUDA_INCLUDE, "cuda_runtime.h")):
        pytest.skip("g++ or the CUDA headers not found")
    out_dir = str(out_dir)
    with open(os.path.join(out_dir, "rep_times_fold.inc"), "w") as f:
        f.write(generate(mutation))
    lib = os.path.join(out_dir, "librep_times.so")
    proc = subprocess.run([gxx, "-std=c++17", "-O2", "-Wall", "-shared", "-fPIC", "-I", out_dir, "-I", CSRC,
                           "-I", os.path.join(ROOT, "include"), "-I", CUDA_INCLUDE, HOST, "-o", lib],
                          capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr[-4000:]
    return lib


class Entry(C.Structure):
    _fields_ = [("measured", C.c_uint32), ("status", C.c_int32), ("bad_sizes", C.c_uint32), ("t0_ns", C.c_float),
                ("peak_gbps", C.c_float), ("half_bytes", C.c_uint64), ("digest", C.c_uint64),
                ("ns_min", C.c_float * 24), ("ns_median", C.c_float * 24), ("ns_max", C.c_float * 24),
                ("sum", C.c_uint64 * 24), ("xr", C.c_uint64 * 24)]


U64P = C.POINTER(C.c_uint64)


def _u64(values):
    return (C.c_uint64 * max(len(values), 1))(*values)


class Fold:
    """The library's four functions over records built from Python lists; every call returns the entry as a dict."""

    def __init__(self, lib_path):
        L = self.lib = C.CDLL(lib_path)
        L.rt_dims.restype = C.c_uint32
        self.max_sizes, self.rep_slots = L.rt_dims(0), L.rt_dims(1)
        L.rt_scratch_new.restype = C.c_void_p
        L.rt_scratch_free.argtypes = [C.c_void_p]
        L.rt_scratch_abort.argtypes = [C.c_void_p, C.c_uint32]
        L.rt_scratch_set.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_uint64] * 4
        L.rt_summarize.argtypes = [U64P, U64P, C.POINTER(C.c_int32), C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32,
                                   C.POINTER(Entry)]
        L.rt_ladder_times.argtypes = [C.POINTER(C.c_float), U64P, C.c_uint32, C.c_uint32, C.c_double, C.c_uint32,
                                      C.POINTER(Entry)]
        L.rt_bw_times.argtypes = [C.c_void_p, U64P, C.c_uint32, C.c_uint32, C.c_double, C.c_uint32, C.POINTER(Entry)]
        L.rt_bw_summarize.argtypes = [C.c_void_p, U64P, U64P, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(Entry)]

    @staticmethod
    def _dict(e, n_sizes, checks=False):
        """The ladder fields of the entry, and with checks its bad_sizes and per-size (S, X)."""
        d = {f: getattr(e, f) for f in ("measured", "status", "t0_ns", "peak_gbps", "half_bytes")}
        for f in ("ns_min", "ns_median", "ns_max") + (("sum", "xr") if checks else ()):
            d[f] = list(getattr(e, f))[:n_sizes]
        if checks:
            d["bad_sizes"] = e.bad_sizes
        return d

    def _scratch(self, b):
        """A BwScratch from b: t_rel, t_end, and optionally sum and xr, each [size][rep] with rep 0 the warm-up, and
        abort."""
        s = self.lib.rt_scratch_new()
        assert s
        for k, row in enumerate(b["t_rel"]):
            for r, t in enumerate(row):
                self.lib.rt_scratch_set(s, k, r, t, b["t_end"][k][r], b["sum"][k][r] if "sum" in b else 0,
                                        b["xr"][k][r] if "xr" in b else 0)
        self.lib.rt_scratch_abort(s, b.get("abort", 0))
        return s

    def summarize(self, ns, digest, status, reps, per_rep, want, idx=3):
        e = Entry()
        self.lib.rt_summarize(_u64(ns), _u64(digest), (C.c_int32 * len(status))(*status), reps, per_rep, want, idx,
                              C.byref(e))
        return {"measured": e.measured, "status": e.status, "digest": e.digest, "ns_min": e.ns_min[0],
                "ns_median": e.ns_median[0], "ns_max": e.ns_max[0]}

    def ladder_times(self, ns, sizes, reps, scale, idx=3):
        t = np.zeros((self.max_sizes, 64), np.float32)
        for k, row in enumerate(ns):
            t[k, :len(row)] = row
        e = Entry()
        self.lib.rt_ladder_times(t.ctypes.data_as(C.POINTER(C.c_float)), _u64(sizes), len(sizes), reps, scale, idx,
                                 C.byref(e))
        return self._dict(e, len(sizes))

    def bw_times(self, b, sizes, reps, scale, idx=3):
        s = self._scratch(b)
        try:
            e = Entry()
            timed = self.lib.rt_bw_times(s, _u64(sizes), len(sizes), reps, scale, idx, C.byref(e))
        finally:
            self.lib.rt_scratch_free(s)
        return bool(timed), self._dict(e, len(sizes))

    def bw_summarize(self, b, want, sizes, reps, idx=3):
        s = self._scratch(b)
        try:
            e = Entry()
            self.lib.rt_bw_summarize(s, _u64([v for sx in want for v in sx]), _u64(sizes), len(sizes), reps, idx,
                                     C.byref(e))
        finally:
            self.lib.rt_scratch_free(s)
        return self._dict(e, len(sizes), checks=True)


# ---- the restatements -----------------------------------------------------------------------------------------------
def f32(v):
    """float32 of a number, rounded once to nearest-even as a C cast from uint64 or double rounds it."""
    if isinstance(v, int):
        assert 0 <= v < 1 << 53, v  # exact in a double, so the cast through it rounds once
        v = float(v)
    return float(np.float32(v))


def ladder_times(ns, sizes, reps, scale):
    """Per size the min, median (element reps // 2 of the sorted reps) and max; t0 the smallest size's median;
    rate scale x size / median (0 for a median of 0); peak the largest rate, rounded to float32 only at the end;
    half the first size whose rate reaches peak / 2."""
    mins, meds, maxs, rates = [], [], [], []
    for row in ns:
        t = sorted(f32(x) for x in row[:reps])
        mins.append(t[0])
        meds.append(t[reps // 2])
        maxs.append(t[-1])
        rates.append(scale * sizes[len(rates)] / meds[-1] if meds[-1] > 0 else 0.0)
    peak = max(rates)
    half = next(s for s, r in zip(sizes, rates) if r >= peak / 2)
    return {"measured": 0, "status": 0, "t0_ns": meds[0], "peak_gbps": f32(peak), "half_bytes": half, "ns_min": mins,
            "ns_median": meds, "ns_max": maxs}


def bw_times(b, sizes, reps, scale):
    """(timed, entry): an aborted kernel gives TIMEOUT and no times; otherwise rep r of size k (r = 1 .. reps) lasted
    t_end[k][r] - t_rel[k][r] ns (uint64 arithmetic), and the warm-up rep 0 counts for nothing."""
    n = len(sizes)
    if b.get("abort", 0):
        return False, {"measured": 1, "status": ERR_TIMEOUT, "t0_ns": 0.0, "peak_gbps": 0.0, "half_bytes": 0,
                       "ns_min": [0.0] * n, "ns_median": [0.0] * n, "ns_max": [0.0] * n}
    ns = [[(b["t_end"][k][r] - b["t_rel"][k][r]) % (1 << 64) for r in range(1, reps + 1)] for k in range(n)]
    return True, dict(ladder_times(ns, sizes, reps, scale), measured=1)


def bw_summarize(b, want, sizes, reps):
    """bw_times at scale 1, then: bit k of bad_sizes when any rep of size k, warm-up included, has an (S, X) other
    than want[k]; (S, X) of the last timed rep; INTEGRITY when a size is bad.  No times and no checks on TIMEOUT."""
    timed, e = bw_times(b, sizes, reps, 1.0)
    n = len(sizes)
    e.update(bad_sizes=0, sum=[0] * n, xr=[0] * n)
    if not timed:
        return e
    for k in range(n):
        if any((b["sum"][k][r], b["xr"][k][r]) != tuple(want[k]) for r in range(reps + 1)):
            e["bad_sizes"] |= 1 << k
        e["sum"][k], e["xr"][k] = b["sum"][k][reps], b["xr"][k][reps]
    e["status"] = ERR_INTEGRITY if e["bad_sizes"] else 0
    return e


def summarize(ns, digest, status, reps, per_rep, want):
    """The digest xors every rep that ran, warm-up included, up to and with the first TIMEOUT rep, which leaves the
    entry TIMEOUT with no times.  Otherwise the last other non-zero status is kept, the times are ns / per_rep of reps
    1 .. reps (the division in double), and a digest other than want is INTEGRITY."""
    d, s = 0, 0
    for k in range(reps + 1):
        d ^= digest[k]
        if status[k] == ERR_TIMEOUT:
            return {"measured": 1, "status": ERR_TIMEOUT, "digest": d, "ns_min": 0.0, "ns_median": 0.0, "ns_max": 0.0}
        if status[k] != 0:
            s = status[k]
    t = sorted(f32(float(ns[k]) / per_rep) for k in range(1, reps + 1))
    return {"measured": 1, "status": ERR_INTEGRITY if d != want else s, "digest": d, "ns_min": t[0],
            "ns_median": t[reps // 2], "ns_max": t[-1]}
