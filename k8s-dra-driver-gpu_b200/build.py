"""Builds libcdprobe.so (sm_90a only) in-tree with nvcc.

The library is the product: hand-written CUDA kernels + the C++ host runtime
behind include/cdprobe.h.  It links the static CUDA runtime and reaches
libcuda.so.1 lazily, so it loads (and every ABI symbol resolves) on a box
without a GPU; cdprobe_open() then fails loudly with CDPROBE_ERR_NO_DEVICE.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libcdprobe.so")
DAEMON = os.path.join(HERE, "cdprobe-daemon")
SOURCES = ["probe_kernels.cu", "bwcurve_kernels.cu", "allreduce_kernels.cu", "allreduce_twoshot_kernels.cu", "allreduce_ll_kernels.cu", "allreduce_ring_kernels.cu", "allreduce_push_kernels.cu", "allreduce_nvls_kernels.cu", "alltoall_kernels.cu", "diagnose_kernels.cu", "latency_kernels.cu", "pingpong_kernels.cu", "atomics_kernels.cu", "handle.cc", "measure.cc", "plan.cc", "schedule.cc", "rendezvous.cc", "vmm.cc", "topo.cc", "links.cc"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=hidden,-Wall,-Wno-unknown-pragmas",
    "-cudart", "static", "-shared",
]


def nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found; libcdprobe.so has no non-CUDA build")
    return exe


def sources() -> list[str]:
    return [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def needs_build() -> bool:
    if not os.path.exists(LIB) or not os.path.exists(DAEMON):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps.append(os.path.join(HERE, "..", "include", "cdprobe.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    cmd = [nvcc(), *NVCC_FLAGS]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    cmd += ["-x", "cu", *sources(), "-o", LIB + ".tmp", "-lpthread", "-ldl", "-lrt"]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + proc.stdout + proc.stderr)
    if verbose:
        sys.stderr.write(proc.stdout + proc.stderr)
    os.replace(LIB + ".tmp", LIB)
    # the daemon mirror (host-only C++, no CUDA): cdprobe-daemon {run,check}
    gxx = shutil.which("g++") or "g++"
    dcmd = [gxx, "-O2", "-std=c++17", "-Wall", os.path.join(CSRC, "daemon_main.cc"), "-o", DAEMON + ".tmp", "-ldl"]
    proc = subprocess.run(dcmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("g++ failed:\n" + " ".join(dcmd) + "\n" + proc.stdout + proc.stderr)
    os.replace(DAEMON + ".tmp", DAEMON)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
