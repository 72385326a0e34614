"""allreduce_nvls_kernel with its two multicast instructions emulated, so that it runs as n ranks on one device.

The product kernel (csrc/allreduce_nvls_kernels.cu) is read when a test asks for it.  Its one multimem.ld_reduce
statement and its one multimem.st statement are replaced by calls to the unicast helpers of tests/c/nvls_emulate.cuh,
and nothing else changes: generate() checks both, so an edit to the kernel either reaches this copy or fails loudly.
build() compiles the copy with the host harness tests/c/nvls_emulate_host.cu into one shared library.

Every rank's kernel must be resident at once, each on its own stream.  Beyond CUDA_DEVICE_MAX_CONNECTIONS streams
(default 8) share hardware queues, and a rank queued behind another would wait for it at the first domain barrier, so
the library runs in a child process with 32 queues (Remote, which talks to `python nvls_emulate.py serve <lib>`).

MUTATIONS are deliberate one-line errors in the copy, each keeping every address inside the allocations, for checking
that the tests see them: build(mutation=name) applies one; test_allreduce_nvls_emulated_gpu.py reads the name from
NVLS_EMULATE_MUTATION."""
import ctypes as C
import difflib
import json
import os
import re
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "k8s-dra-driver-gpu_b200", "csrc")
KERNEL = os.path.join(CSRC, "allreduce_nvls_kernels.cu")
HEADER = os.path.join(HERE, "c", "nvls_emulate.cuh")
HOST = os.path.join(HERE, "c", "nvls_emulate_host.cu")
NO_FAULT = 0xFFFFFFFF  # kArNoFault

LD_REDUCE = re.compile(r'asm volatile\("multimem\.ld_reduce\.relaxed\.sys\.global\.add\.u64 %0, \[%1\];" : "=l"\(v\) '
                       r': "l"\(mc\) : "memory"\);')
LD_REDUCE_CALL = "v = nvls_emul_ld_reduce(mc);"
STORE = re.compile(r'asm volatile\("multimem\.st\.relaxed\.sys\.global\.v4\.f32 \[%0\], \{%1, %2, %3, %4\};"[^;]*?'
                   r': "memory"\);', re.S)
STORE_CALL = "nvls_emul_st(mc, w0, w1);"

# name: (text in the generated copy, its replacement); each text occurs exactly once.  What each one breaks, and the
# test of test_allreduce_nvls_emulated_gpu.py that fails under it:
#   walk_drops_last_unit              the last unit of every chunk is never stored: test_clean_ladders_on_every_grid
#   fault_halves_swapped              the fault lands on the other word of its vector: the (vec, vec + 1) places of
#                                     test_each_fault_fails_exactly_the_words_the_restatement_names
#   fault_every_rep                   the fault acts in every rep: the same test at reps = 3
#   partial_unit_last_vector_skipped  a partial unit's last 16 bytes are never stored: test_clean_ladders_on_every_grid
#   second_word_from_first            every odd word holds the even word's sum: test_clean_ladders_on_every_grid
# A rotation of the chunk owners is not among them: every unit is still reduced and stored once, so the clean checks
# cannot see it.
MUTATIONS = {
    "walk_drops_last_unit": ("Walk<false>{hi, lo + gwarp, 0ull, nwarps, nullptr}",
                             "Walk<false>{hi > lo ? hi - 1 : hi, lo + gwarp, 0ull, nwarps, nullptr}"),
    "fault_halves_swapped": ("if (fb & 8u) w1 ^= 1ull;\n        else w0 ^= 1ull;",
                             "if (fb & 8u) w0 ^= 1ull;\n        else w1 ^= 1ull;"),
    "fault_every_rep": ("(r == 1u && k == P.fault_k)", "(k == P.fault_k)"),
    "partial_unit_last_vector_skipped": ("if (off >= len) continue;\n      uint64_t w0",
                                         "if (off >= len || (len < kUnitBytes && off + 16 >= len)) continue;\n"
                                         "      uint64_t w0"),
    "second_word_from_first": ("mc_ld_reduce_add_u64(in + off + 8)", "mc_ld_reduce_add_u64(in + off)"),
}


def generate(text=None, mutation=None):
    """The kernel source with its two multimem statements replaced (and `mutation` applied).  Asserts that each
    statement occurs exactly once and that the copy differs from the product file in those two statements only."""
    if text is None:
        with open(KERNEL) as f:
            text = f.read()
    out, n_ld = LD_REDUCE.subn(LD_REDUCE_CALL, text)
    out, n_st = STORE.subn(STORE_CALL, out)
    assert (n_ld, n_st) == (1, 1), f"multimem.ld_reduce matched {n_ld} times, multimem.st {n_st} times"
    diff = list(difflib.ndiff(text.splitlines(), out.splitlines()))
    removed = [l[2:].strip() for l in diff if l.startswith("- ")]
    added = [l[2:].strip() for l in diff if l.startswith("+ ")]
    statements = LD_REDUCE.findall(text) + STORE.findall(text)
    assert " ".join(removed) == " ".join(" ".join(s.split()) for s in statements), removed
    assert added == [LD_REDUCE_CALL, STORE_CALL], added
    if mutation is not None:
        old, new = MUTATIONS[mutation]
        assert out.count(old) == 1, (mutation, out.count(old))
        out = out.replace(old, new)
    return out


def nvcc():
    """Path of nvcc, or None."""
    import shutil

    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return exe if os.path.exists(exe) else None


def build(out_dir, mutation=None, ptxas_verbose=False):
    """Compiles the emulated copy with the host harness into out_dir/libnvls_emulate.so; returns (its path, nvcc's
    stderr).  Skips the calling test when nvcc is missing."""
    import pytest

    exe = nvcc()
    if exe is None:
        pytest.skip("nvcc not found")
    out_dir = str(out_dir)
    with open(os.path.join(out_dir, "allreduce_nvls_emulated.cu"), "w") as f:
        f.write(generate(mutation=mutation))
    lib = os.path.join(out_dir, "libnvls_emulate.so")
    proc = subprocess.run([exe, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", CSRC,
                           "-I", out_dir, "-include", HEADER, "-shared", "-Xcompiler", "-fPIC",
                           *(["-Xptxas", "-v"] if ptxas_verbose else []), HOST, "-o", lib],
                          capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr[-4000:]
    return lib, proc.stderr


class Emulator:
    """The harness library in this process."""

    def __init__(self, lib_path):
        L = self.lib = C.CDLL(lib_path)
        L.nvls_emul_open.restype = C.c_void_p
        L.nvls_emul_open.argtypes = [C.c_uint32, C.POINTER(C.c_uint32), C.c_uint64, C.c_uint64]
        L.nvls_emul_call.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.c_uint32, C.c_uint32, C.c_int32, C.c_uint32,
                                     C.c_uint32, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64)]
        L.nvls_emul_corrupt.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint64]
        L.nvls_emul_close.argtypes = [C.c_void_p]
        L.nvls_emul_error.restype = C.c_char_p
        dims = (C.c_uint64 * 3)()
        L.nvls_emul_dims(dims)
        self.S, self.R, self.row_words = dims
        self.ctx = {}

    def _err(self, what):
        raise RuntimeError(f"{what}: {self.lib.nvls_emul_error().decode()}")

    def device(self):
        v = (C.c_uint64 * 3)()
        if self.lib.nvls_emul_device(v) != 0:
            self._err("device")
        return {"sms": v[0], "free": v[1], "total": v[2]}

    def open(self, n, grids, s_max, seed):
        h = self.lib.nvls_emul_open(n, (C.c_uint32 * n)(*grids), s_max, seed)
        if not h:
            self._err("open")
        self.ctx[h] = n
        return h

    def call(self, h, sizes, reps, fault=None, fault_rank=-1, call_seq=1):
        """Every rank's row: sum, xr, t_rel, t_end [size][rep] (rep 0: the warm-up), bad_words and first_bad [size],
        abort.  fault (mode, k, word) goes to fault_rank, or to the word's owner when fault_rank < 0."""
        n, ns = self.ctx[h], len(sizes)
        rows = np.zeros(n * self.row_words, np.uint64)
        mode, k, word = fault if fault is not None else (0, NO_FAULT, 0)
        rc = self.lib.nvls_emul_call(h, (C.c_uint64 * ns)(*sizes), ns, reps, fault_rank, mode, k, word, call_seq,
                                     rows.ctypes.data_as(C.POINTER(C.c_uint64)))
        if rc != 0:
            self._err("call")
        out = []
        SR = self.S * self.R
        for row in rows.reshape(n, self.row_words):
            def rep_table(i):
                return [[int(v) for v in r[:reps + 1]] for r in row[i * SR:(i + 1) * SR].reshape(self.S, self.R)[:ns]]
            out.append({"sum": rep_table(0), "xr": rep_table(1), "t_rel": rep_table(2), "t_end": rep_table(3),
                        "bad_words": [int(v) for v in row[4 * SR:4 * SR + ns]],
                        "first_bad": [int(v) for v in row[4 * SR + self.S:4 * SR + self.S + ns]],
                        "abort": int(row[4 * SR + 2 * self.S])})
        return out

    def corrupt(self, h, rank, word, mask):
        if self.lib.nvls_emul_corrupt(h, rank, word, mask) != 0:
            self._err("corrupt")

    def close(self, h):
        self.lib.nvls_emul_close(h)
        del self.ctx[h]


def serve(lib_path):
    """Answers one JSON request per input line, {"op": method, "args": [...]}, with one JSON line: {"ok": result} or
    {"error": text}."""
    emu = Emulator(lib_path)
    for line in sys.stdin:
        req = json.loads(line)
        try:
            res = {"ok": getattr(emu, req["op"])(*req["args"])}
        except Exception as e:  # reported to the test, which fails with it
            res = {"error": f"{type(e).__name__}: {e}"}
        sys.stdout.write(json.dumps(res) + "\n")
        sys.stdout.flush()


class Remote:
    """An Emulator in a child process with CUDA_DEVICE_MAX_CONNECTIONS=32, so that up to 16 ranks' streams each get a
    hardware queue of their own.  Same methods; a context handle is an int."""

    def __init__(self, lib_path):
        env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
        self.proc = subprocess.Popen([sys.executable, os.path.abspath(__file__), "serve", lib_path], env=env,
                                     stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)

    def _ask(self, op, *args):
        self.proc.stdin.write(json.dumps({"op": op, "args": list(args)}) + "\n")
        self.proc.stdin.flush()
        line = self.proc.stdout.readline()
        assert line, f"the emulator process ended (exit {self.proc.wait()})"
        res = json.loads(line)
        if "error" in res:
            raise RuntimeError(res["error"])
        return res["ok"]

    def device(self):
        return self._ask("device")

    def open(self, n, grids, s_max, seed):
        return self._ask("open", n, list(grids), s_max, seed)

    def call(self, h, sizes, reps, fault=None, fault_rank=-1, call_seq=1):
        return self._ask("call", h, list(sizes), reps, list(fault) if fault else None, fault_rank, call_seq)

    def corrupt(self, h, rank, word, mask):
        return self._ask("corrupt", h, rank, word, mask)

    def close(self, h):
        return self._ask("close", h)

    def shutdown(self):
        self.proc.stdin.close()
        self.proc.wait(timeout=60)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.shutdown()


if __name__ == "__main__":
    assert sys.argv[1] == "serve"
    serve(sys.argv[2])
