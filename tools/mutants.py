"""Runs the mutant catalogue of tests/mutants.py on a GPU: for every mutant, a fresh copy of the tracked tree with the
mutant applied, its own libcdprobe.so built there, and `pytest -m gpu -x -q <the mutant's killers>` run in it.  A
mutant is killed when a killer fails.  First the unmutated tree runs every killer of the selection, once: a killer
that fails there would count any mutant as killed, so the run stops.  Prints one JSON document (also to --out): per
mutant, killed or survived, the first failing test, the build and test wall times.

The copies live in a temporary directory and are deleted as soon as their tests end; the working tree is only read.
Builds run ahead of the tests, up to --jobs at once (CPU work only), and the tests of one mutant at a time, so no two
GPU processes overlap and each ends before the next mutant starts.  The tracked tree is `git ls-files`; where the tree
is not a git checkout, every file that .gitignore does not exclude.

  python tools/mutants.py [--only NAME ...] [--jobs N] [--out FILE]"""
import argparse
import concurrent.futures as cf
import fnmatch
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mutants as M  # noqa: E402

BUILD_TIMEOUT_S = 900
TEST_TIMEOUT_S = 1200
# Runs pytest in the copy and then names every libcdprobe.so the process has mapped, so the runner can check that the
# tests loaded the copy's own library.
PYTEST = ("import sys, pytest\n"
          "rc = pytest.main(sys.argv[1:])\n"
          "maps = sorted({l.split()[-1] for l in open('/proc/self/maps') if l.rstrip().endswith('libcdprobe.so')})\n"
          "print('MAPPED ' + ' '.join(maps))\n"
          "sys.exit(int(rc))\n")


def tracked_files():
    """Paths, relative to ROOT, of the files the copy gets."""
    try:
        out = subprocess.run(["git", "ls-files", "-z"], cwd=ROOT, capture_output=True, check=True).stdout
        return [p for p in out.decode().split("\0") if p and os.path.isfile(os.path.join(ROOT, p))]
    except (OSError, subprocess.CalledProcessError):
        pass
    patterns = []
    with open(os.path.join(ROOT, ".gitignore")) as f:
        patterns = [l.strip() for l in f if l.strip() and not l.startswith("#")]

    def ignored(rel, is_dir):
        for p in patterns:
            if p.endswith("/") and not is_dir:
                continue
            p = p.rstrip("/")
            if ("/" in p and fnmatch.fnmatch(rel, p.lstrip("/"))) or fnmatch.fnmatch(os.path.basename(rel), p):
                return True
        return False

    files = []
    for d, dirs, names in os.walk(ROOT):
        rel_d = os.path.relpath(d, ROOT)
        dirs[:] = [x for x in dirs if x != ".git" and not ignored(os.path.normpath(os.path.join(rel_d, x)), True)]
        files += [os.path.normpath(os.path.join(rel_d, n)) for n in names
                  if not ignored(os.path.normpath(os.path.join(rel_d, n)), False)]
    return sorted(files)


def prepare(m, files):
    """A fresh copy of the tree with m applied (none: unmutated) and its library built: (copy, build seconds, build
    error or None)."""
    copy = tempfile.mkdtemp(prefix=f"cdprobe-mutant-{m['name']}-")
    for rel in files:
        dst = os.path.join(copy, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copy2(os.path.join(ROOT, rel), dst)
    if m["file"] is not None:
        text = M.mutated(m, copy)
        with open(os.path.join(copy, "k8s-dra-driver-gpu_b200", "csrc", m["file"]), "w") as f:
            f.write(text)
    t0 = time.monotonic()
    # the same entry point the suite's pkg fixture calls; it finds the library up to date and does not rebuild
    proc = subprocess.run([sys.executable, "-c", "import __graft_entry__ as g; g.build()"], cwd=copy,
                          capture_output=True, text=True, timeout=BUILD_TIMEOUT_S)
    err = None if proc.returncode == 0 else (proc.stdout + proc.stderr)[-2000:]
    return copy, time.monotonic() - t0, err


def run_tests(m, copy, stop_first=True):
    """Runs m's killers in the copy: (rc, first failing test or None, mapped libcdprobe.so paths, seconds, tail)."""
    assert not any("test_sass_pins_cpu.py" in k for k in m["killers"]), m["name"]
    t0 = time.monotonic()
    cmd = [sys.executable, "-c", PYTEST, "-m", "gpu", *(["-x"] if stop_first else []), "-q", "-rfE",
           "-p", "no:cacheprovider", *m["killers"]]
    proc = subprocess.Popen(cmd, cwd=copy, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                            start_new_session=True)
    try:
        out, _ = proc.communicate(timeout=TEST_TIMEOUT_S)
    except subprocess.TimeoutExpired:
        os.killpg(proc.pid, 9)
        out, _ = proc.communicate()
        out += f"\n(no result within {TEST_TIMEOUT_S} s)"
    failed = re.findall(r"^(?:FAILED|ERROR) (\S+)", out, re.M)
    mapped = re.findall(r"^MAPPED (.*)$", out, re.M)
    return proc.returncode, failed[0] if failed else None, mapped[-1].split() if mapped else [], \
        time.monotonic() - t0, out[-3000:]


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--only", nargs="*", help="run these mutants only")
    ap.add_argument("--jobs", type=int, default=os.cpu_count() or 1, help="builds in flight at once")
    ap.add_argument("--out", help="also write the JSON document here")
    args = ap.parse_args()
    todo = [M.by_name(n) for n in args.only] if args.only else list(M.MUTANTS)
    files = tracked_files()
    t_start = time.monotonic()
    rows = []
    baseline = {"name": "unmutated", "file": None, "killers": sorted({k for m in todo for k in m["killers"]})}
    with cf.ThreadPoolExecutor(max_workers=max(1, args.jobs)) as pool:
        builds = [pool.submit(prepare, m, files) for m in [baseline] + todo]
        copy, build_s, err = builds[0].result()
        try:
            assert err is None, err
            rc, first, mapped, test_s, tail = run_tests(baseline, copy, stop_first=False)
        finally:
            shutil.rmtree(copy, ignore_errors=True)
        print(f"unmutated: pytest exit {rc} over {len(baseline['killers'])} killers in {test_s:.0f} s",
              file=sys.stderr, flush=True)
        if rc != 0:
            for fut in builds[1:]:
                fut.cancel()
            for fut in builds[1:]:
                if not fut.cancelled():
                    shutil.rmtree(fut.result()[0], ignore_errors=True)
            sys.stderr.write(tail + "\n")
            print(json.dumps({"unmutated": {"result": f"pytest exit {rc}", "first_failure": first, "detail": tail}}))
            return 2
        unmutated = {"test_s": round(test_s, 1), "killers": len(baseline["killers"]), "result": "passed"}
        for m, fut in zip(todo, builds[1:]):
            copy, build_s, err = fut.result()
            row = {"name": m["name"], "file": m["file"], "build_s": round(build_s, 1)}
            try:
                if err is not None:
                    row.update(result="build failed", detail=err)
                else:
                    rc, first, mapped, test_s, tail = run_tests(m, copy)
                    own = os.path.join(os.path.realpath(copy), "k8s-dra-driver-gpu_b200", "libcdprobe.so")
                    assert all(os.path.realpath(p) == own for p in mapped), (m["name"], mapped)
                    row.update(test_s=round(test_s, 1), loaded_own_library=bool(mapped), first_failure=first,
                               result="killed" if rc == 1 and first else "survived" if rc == 0 else f"pytest exit {rc}")
                    if row["result"] != "killed":
                        row["detail"] = tail
            finally:
                shutil.rmtree(copy, ignore_errors=True)
            row["listed_killer"] = bool(row.get("first_failure")) and \
                any(row["first_failure"] == k or row["first_failure"].startswith(k + "[") for k in m["killers"])
            rows.append(row)
            print(f"{m['name']}: {row['result']} {row.get('first_failure') or ''} "
                  f"(build {row['build_s']} s, tests {row.get('test_s', '-')} s)", file=sys.stderr, flush=True)
    doc = {"unmutated": unmutated, "mutants": rows, "killed": sum(r["result"] == "killed" for r in rows),
           "total": len(rows),
           "wall_s": round(time.monotonic() - t_start, 1), "jobs": args.jobs}
    text = json.dumps(doc, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")
    return 0 if doc["killed"] == doc["total"] else 1


if __name__ == "__main__":
    sys.exit(main())
