"""Plumbing the tests share: values and struct layouts that gcc computes from include/cdprobe.h, the C helpers under
tests/c, the symbols the header declares and the library exports, a Probe over a fake library, and one child process per
rank of a domain.  exported_symbols skips the calling test when nm is missing."""
import contextlib
import ctypes as C
import json
import os
import re
import shutil
import subprocess
import sys
import uuid

import pytest

from conftest import ROOT
from kernel_tools import CSRC

HEADER = os.path.join(ROOT, "include", "cdprobe.h")


def header_values(tmp_path, *exprs):
    """The value of each C expression (a macro, or a sizeof/offsetof) over include/cdprobe.h, as a program built by gcc
    prints it, in the order given."""
    body = "".join(f'printf("%llu\\n", (unsigned long long)({e}));' for e in exprs)
    src = tmp_path / "values.c"
    src.write_text(f'#include <stddef.h>\n#include <stdio.h>\n#include "{HEADER}"\nint main(void){{{body} return 0;}}\n')
    exe = tmp_path / "values"
    subprocess.run(["gcc", "-o", str(exe), str(src)], check=True)
    return [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]


def assert_layout(tmp_path, structs):
    """Asserts that gcc's sizeof and offsetof of every field of each C struct equal its ctypes mirror's, for
    {C type name: ctypes structure}."""
    checks = []
    for cname, ct in structs.items():
        checks.append((f"sizeof({cname})", C.sizeof(ct), cname))
        checks += [(f"offsetof({cname}, {f})", getattr(ct, f).offset, f"{cname}.{f}") for f, _ in ct._fields_]
    for got, (_, want, what) in zip(header_values(tmp_path, *(e for e, _, _ in checks)), checks):
        assert got == want, what


def c_tool_exe(tmp_path_factory, source, opt="-O2", csrc=()):
    """Path of tests/c/<source> built by g++ against the library's csrc/ headers, linked with the csrc/ files named."""
    exe = tmp_path_factory.mktemp(os.path.splitext(source)[0]) / os.path.splitext(source)[0]
    subprocess.run(["g++", "-std=c++17", opt, "-Wall", "-I", CSRC, os.path.join(ROOT, "tests", "c", source),
                    *(os.path.join(CSRC, f) for f in csrc), "-o", str(exe)], check=True)
    return str(exe)


def c_tool(tmp_path_factory, source, opt="-O2"):
    """run(lines) over tests/c/<source> built as c_tool_exe builds it: feeds it one input line per entry (a string, or
    a sequence of values joined by spaces) and returns the integer columns of its one output line per input line."""
    exe = c_tool_exe(tmp_path_factory, source, opt)

    def run(lines):
        text = "".join((l if isinstance(l, str) else " ".join(str(x) for x in l)) + "\n" for l in lines)
        out = subprocess.run([exe], input=text, capture_output=True, text=True, check=True).stdout.splitlines()
        assert len(out) == len(lines)
        return [[int(x) for x in l.split()] for l in out]

    return run


def declared_symbols():
    """The names of the functions include/cdprobe.h declares with CDPROBE_API."""
    return set(re.findall(r"CDPROBE_API\s+[\w\s\*]+?\b(cdprobe_\w+)\s*\(", open(HEADER).read()))


def exported_symbols(lib_path):
    """The names of the dynamic symbols the shared library `lib_path` defines, as nm reads them."""
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not found")
    out = subprocess.run([nm, "-D", "--defined-only", lib_path], capture_output=True, text=True, check=True).stdout
    return {l.split()[-1] for l in out.splitlines() if l.strip()}


class FakeLib:
    """The error-text entry points a Probe reads when a fake library's call fails; a test's subclass adds the entry
    point it fakes."""

    def cdprobe_strerror(self, rc):
        return b"invalid argument"

    def cdprobe_last_error(self):
        return b""


@contextlib.contextmanager
def fake_probe(pkg, lib):
    """A Probe whose calls go to `lib` with the handle 0x1234, without opening one; the handle is cleared on exit so
    that closing the Probe calls nothing."""
    p = object.__new__(pkg.Probe)
    p._lib, p._h = lib, C.c_void_p(0x1234)
    try:
        yield p
    finally:
        p._h = C.c_void_p()


def run_children(script, world, *argv, timeout=600):
    """Runs the Python `script` in one process per rank of a new rendezvous session, with the arguments session, rank,
    world and `argv`; asserts that each exits 0 and returns the JSON of each one's last `RESULT ` line, in rank order."""
    session = f"t-{uuid.uuid4().hex[:12]}"
    procs = [subprocess.Popen([sys.executable, "-c", script, session, str(r), str(world), *(str(a) for a in argv)],
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for r in range(world)]
    outs = []
    for pr in procs:
        so, se = pr.communicate(timeout=timeout)
        assert pr.returncode == 0, se[-2000:]
        outs.append(json.loads([l for l in so.splitlines() if l.startswith("RESULT ")][-1][7:]))
    return outs
