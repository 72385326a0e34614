"""What the CUDA tools report about the compiled kernels, for the tests that check them: ptxas's resource report of one
translation unit, one kernel's SASS in the built library, and the pins of every function's SASS.  Each skips the
calling test when its tool is missing."""
import functools
import hashlib
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "k8s-dra-driver-gpu_b200", "csrc")


def _tool(name):
    exe = shutil.which(name) or os.path.join("/usr/local/cuda/bin", name)
    if not os.path.exists(exe):
        pytest.skip(f"{name} not found")
    return exe


@functools.cache
def _ptxas(nvcc, unit):
    with tempfile.TemporaryDirectory() as tmp:
        proc = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                               "-c", os.path.join(CSRC, unit), "-o", os.path.join(tmp, "k.o")],
                              capture_output=True, text=True, check=True)
    found = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", proc.stderr)
    return tuple((name, tuple(int(v) for v in vals)) for name, *vals in found)


def ptxas_report(unit):
    """{mangled function: (stack frame, spill stores, spill loads), in bytes} as ptxas -v reports them when csrc/<unit>
    is compiled alone with the build's device flags."""
    return dict(_ptxas(_tool("nvcc"), unit))


@functools.cache
def _sass(cuobjdump, lib):
    out = subprocess.run([cuobjdump, "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for f in re.split(r"\n\s*Function : ", out)[1:]:
        name, body = f.split("\n", 1)
        ins = re.findall(r"/\*([0-9a-f]{4,})\*/\s+([^;]*);", body)
        funcs[name.strip()] = ([int(a, 16) for a, _ in ins], [t.strip() for _, t in ins])
    return funcs


def kernel_sass(lib, pattern):
    """(addresses, instructions) of the one function in the library `lib` whose mangled name matches the regular
    expression `pattern` (re.search)."""
    funcs = _sass(_tool("cuobjdump"), lib)
    names = [n for n in funcs if re.search(pattern, n)]
    assert len(names) == 1, (pattern, names)
    addr, text = funcs[names[0]]
    return list(addr), list(text)


def sass_pins(lib):
    """{function: [instruction count, sha256 of the instructions joined by newlines]} for every function in the library
    `lib`, as kernel_sass reads them.  A function in an anonymous namespace is keyed without the two hashes nvcc puts
    in that namespace's name, which change with the build directory."""
    pins = {}
    for name, (_, text) in _sass(_tool("cuobjdump"), lib).items():
        key = re.sub(r"_GLOBAL__N__[0-9a-f]{8}_(\w+?_cu)_[0-9a-f]{8}", r"_GLOBAL__N__\1", name)
        pins[key] = [len(text), hashlib.sha256("\n".join(text).encode()).hexdigest()]
    return pins
