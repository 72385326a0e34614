"""The mutant catalogue of tests/mutants.py, checked without a GPU: every entry applies exactly once inside its named
function, changes something, keeps to the safety rule and compiles for sm_90a; names are unique; every listed killer
is a GPU test of the collected suite; every kernel unit and shared header has entries; and an anchor that no longer
matches fails loudly.  tools/mutants.py runs the catalogue on a GPU."""
import concurrent.futures as cf
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

import pytest

import mutants as M

KERNEL_FILES = ["probe_kernels.cu", "diagnose_kernels.cu", "latency_kernels.cu", "pingpong_kernels.cu",
                "atomics_kernels.cu", "bwcurve_kernels.cu", "alltoall_kernels.cu", "allreduce_kernels.cu",
                "allreduce_twoshot_kernels.cu", "allreduce_ll_kernels.cu", "allreduce_ring_kernels.cu",
                "allreduce_push_kernels.cu", "allreduce_nvls_kernels.cu", "datapath.cuh", "allreduce_path.cuh",
                "timed_rep.cuh", "measure.cc"]
IDS = [m["name"] for m in M.MUTANTS]


def test_names_are_unique_and_the_catalogue_covers_every_kernel_file():
    assert len(set(IDS)) == len(IDS), sorted(n for n in IDS if IDS.count(n) > 1)
    assert all(re.fullmatch(r"[a-z0-9_]+", n) for n in IDS)
    per_file = {f: sum(m["file"] == f for m in M.MUTANTS) for f in KERNEL_FILES}
    assert all(n >= 2 for n in per_file.values()), per_file
    assert {m["file"] for m in M.MUTANTS} == set(KERNEL_FILES)
    assert len(M.MUTANTS) >= 50
    assert any(m["function"] == "fold_checks" for m in M.MUTANTS)
    assert set(M.KILLED_BY) == set(IDS)


@pytest.mark.parametrize("m", M.MUTANTS, ids=IDS)
def test_the_anchor_applies_once_inside_its_function_and_keeps_to_the_safety_rule(m):
    with open(os.path.join(M.CSRC, m["file"])) as f:
        text = f.read()
    assert m["old"] != m["new"]
    start, end = M.body(text, m["function"])
    assert text[start:end].count(m["old"]) == 1, (m["name"], text[start:end].count(m["old"]))
    out = M.apply(text, m)
    assert out != text and out[:start] == text[:start] and out.endswith(text[end:])
    assert M.safety_problems(m) == [], (m["name"], M.safety_problems(m))
    assert m["killers"] and all(k.startswith("tests/test_") and "::" in k for k in m["killers"]), m["killers"]
    assert not any("test_sass_pins_cpu.py" in k for k in m["killers"])
    # every mutant was killed on the last GPU run, by one of its listed killers
    assert m["killed_by"] is not None and (m["killed_by"] in m["killers"] or
                                           any(m["killed_by"].startswith(k + "[") for k in m["killers"])), \
        (m["name"], m["killed_by"])


def test_a_changed_anchor_fails_loudly():
    m = M.by_name("fold_unit_neighbour_granule")
    with open(os.path.join(M.CSRC, m["file"])) as f:
        text = f.read()
    # the anchor edited away, or present twice
    for broken in (text.replace(m["old"], "rotl64(unit_xor, fold6(g + 0))"),
                   M.replace_once(text, m["old"], m["old"] + "; (void)" + m["old"], "datapath.cuh")):
        with pytest.raises(AssertionError, match="occurs"):
            M.apply(broken, m)
    # the anchor text outside the named function only
    moved = text.replace(m["old"], "rotl64(unit_xor, 0)").replace("uint64_t left = bytes",
                                                                    "uint64_t left = " + m["old"] + " * 0 + bytes")
    with pytest.raises(AssertionError, match="occurs 0 times"):
        M.apply(moved, m)
    # the function renamed, or defined twice
    with pytest.raises(AssertionError, match="0 definitions"):
        M.apply(text.replace("void fold_unit(", "void fold_granule("), m)
    with pytest.raises(AssertionError, match="2 definitions"):
        M.body(text + "\nvoid fold_unit(int) { }\n", "fold_unit")


def test_the_safety_rule_refuses_walks_waits_and_addresses():
    def problems(old, new):
        return M.safety_problems({"old": old, "new": new})

    assert problems("for (uint32_t r = 0; r <= P.reps; ++r)", "for (uint32_t r = 0; r < P.reps; ++r)")
    assert problems("spin_until<kScopeGpu>(c, &lb->written.v, n_units)", "spin_until<kScopeGpu>(c, &lb->written.v, 1)")
    assert problems("stg_pair(base + off, w0, w1);", "stg_pair(base + off + 16, w0, w1);")
    assert problems("acc[2 * i] += 1ull;", "acc[2 * i + 2] += 1ull;")
    assert problems("__threadfence_system();", ";")
    assert problems("x = a;", "x = a; break;")
    assert problems("ux ^= w0 ^ w1;", "ux ^= w0 ^ w1; stg_v4(p, q);")
    assert problems("stg_pair(base + off, w0, w1);", "stg_pair(base + off, w1, w0);") == []


def test_every_killer_is_a_collected_gpu_test():
    proc = subprocess.run([sys.executable, "-m", "pytest", "--collect-only", "-q", "-m", "gpu",
                           "-p", "no:cacheprovider", "tests"], cwd=M.ROOT, capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout[-3000:] + proc.stderr[-3000:]
    collected = {l.split("[")[0] for l in proc.stdout.splitlines() if "::" in l}
    missing = sorted({k for m in M.MUTANTS for k in m["killers"]} - collected)
    assert not missing, missing


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return exe if os.path.exists(exe) else None


def test_every_mutated_unit_compiles_for_sm_90a(tmp_path):
    """Each mutant's file, mutated, compiled (-c only) in every unit of libcdprobe.so that includes it, with the
    library's own flags; all compiles in parallel."""
    exe = _nvcc()
    if exe is None:
        pytest.skip("nvcc not found")
    import cdprobe_pkg

    flags = [f for f in cdprobe_pkg.load().build.NVCC_FLAGS if f not in ("-shared", "-cudart", "static", "-lineinfo")]
    jobs = []
    for m in M.MUTANTS:
        tree = tempfile.mkdtemp(prefix=m["name"] + "-", dir=tmp_path)
        shutil.copytree(os.path.join(M.ROOT, "include"), os.path.join(tree, "include"))
        csrc = os.path.join(tree, "k8s-dra-driver-gpu_b200", "csrc")
        shutil.copytree(M.CSRC, csrc)
        with open(os.path.join(csrc, m["file"]), "w") as f:
            f.write(M.mutated(m))
        jobs += [(m["name"], u, [exe, *flags, "-x", "cu", "-c", os.path.join(csrc, u), "-o",
                                 os.path.join(tree, u + ".o")]) for u in M.units(m)]

    def compile_one(job):
        proc = subprocess.run(job[2], capture_output=True, text=True)
        return job[0], job[1], proc.returncode, proc.stderr[-2000:]

    t0 = time.monotonic()
    with cf.ThreadPoolExecutor(max_workers=os.cpu_count() or 1) as pool:
        results = list(pool.map(compile_one, jobs))
    failed = [(n, u, err) for n, u, rc, err in results if rc != 0]
    assert not failed, failed[:3]
    print(f"{len(jobs)} mutated units compiled in {time.monotonic() - t0:.0f} s on {os.cpu_count()} CPUs")
