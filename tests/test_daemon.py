"""`cdprobe-daemon {run,check}` — the fabric-probe slice of cmd/compute-domain-daemon.

`check` must keep the reference's behaviour (cmd/compute-domain-daemon/main.go:435-459): no-op text
when CLIQUE_ID is empty, otherwise `nvidia-imex-ctl -c /imexd/imexd.cfg -q` == "READY\\n"; on top of
that it consults the verdict file `run` writes.  The reference has no unit test for the daemon (SURVEY
§4), so these are written the way its bats tests assert: on exit codes and output text."""
import json
import os
import subprocess

import pytest

from conftest import ROOT, gpu_count

DAEMON = os.path.join(ROOT, "k8s-dra-driver-gpu_b200", "cdprobe-daemon")
LIB = os.path.join(ROOT, "k8s-dra-driver-gpu_b200", "libcdprobe.so")


def daemon(args, env=None, timeout=120):
    e = {"PATH": os.environ.get("PATH", ""), "LD_LIBRARY_PATH": os.environ.get("LD_LIBRARY_PATH", "")}
    e.update(env or {})
    return subprocess.run([DAEMON, *args], env=e, capture_output=True, text=True, timeout=timeout)


def fake_ctl(tmp_path, text, code=0):
    p = tmp_path / "nvidia-imex-ctl"
    p.write_text(f"#!/bin/sh\n[ \"$1\" = -c ] && [ \"$2\" = /imexd/imexd.cfg ] && [ \"$3\" = -q ] || exit 64\nprintf '{text}'\nexit {code}\n")
    p.chmod(0o755)
    return str(p)


@pytest.fixture(autouse=True)
def _built(pkg):
    assert os.path.exists(DAEMON)


def test_check_noop_without_clique(tmp_path):
    r = daemon(["check"], {"CLIQUE_ID": "", "FABRIC_PROBE_VERDICT_PATH": str(tmp_path / "none.json")})
    assert r.returncode == 0
    assert r.stdout == "check succeeded (noop, clique ID is empty)\n"  # main.go:437, byte for byte


def test_check_ready_with_clique(tmp_path):
    r = daemon(["check"], {"CLIQUE_ID": "u.1", "CDPROBE_IMEX_CTL": fake_ctl(tmp_path, "READY\\n"),
                           "FABRIC_PROBE_VERDICT_PATH": str(tmp_path / "none.json")})
    assert r.returncode == 0 and r.stdout == ""


@pytest.mark.parametrize("text,code,needle", [
    ("NOT_READY\\n", 0, "IMEX daemon not ready: NOT_READY"),
    ("READY", 0, "IMEX daemon not ready: READY"),               # missing newline is not READY\n
    ("READY\\nmore\\n", 0, "IMEX daemon not ready"),
    ("READY\\n", 3, "IMEX daemon check failed: error running"),  # non-zero exit fails even with READY
])
def test_check_not_ready_with_clique(tmp_path, text, code, needle):
    r = daemon(["check"], {"CLIQUE_ID": "u.1", "CDPROBE_IMEX_CTL": fake_ctl(tmp_path, text, code),
                           "FABRIC_PROBE_VERDICT_PATH": str(tmp_path / "none.json")})
    assert r.returncode == 1 and needle in r.stderr


def test_check_missing_imex_ctl_fails(tmp_path):
    r = daemon(["check"], {"CLIQUE_ID": "u.1", "CDPROBE_IMEX_CTL": str(tmp_path / "absent"),
                           "FABRIC_PROBE_VERDICT_PATH": str(tmp_path / "none.json")})
    assert r.returncode == 1 and "IMEX daemon check failed" in r.stderr


def verdict(tmp_path, ok, **kw):
    d = {"time_unix": kw.pop("time_unix", 2000000000), "ok": ok, "n": 8, "unreachable_pairs": kw.pop("unreachable", 0),
         "min_gbps_read": 665.0, "min_gbps_write": 690.0, "probe_ms": 3.5, "bytes_per_pair": 153391616, "error": ""}
    d.update(kw)
    p = tmp_path / "fabricprobe.json"
    p.write_text(json.dumps(d, indent=1).replace(": True", ": true"))
    return str(p)


def test_check_consults_probe_verdict(tmp_path):
    env = {"CLIQUE_ID": ""}
    assert daemon(["check"], {**env, "FABRIC_PROBE_VERDICT_PATH": verdict(tmp_path, True)}).returncode == 0
    r = daemon(["check"], {**env, "FABRIC_PROBE_VERDICT_PATH": verdict(tmp_path, False, unreachable=2)})
    assert r.returncode == 1 and "fabric probe failed: 2 unreachable pair(s)" in r.stderr
    # the reference's no-op text is still printed first: the IMEX part of the gate did pass
    assert r.stdout == "check succeeded (noop, clique ID is empty)\n"
    # a stale verdict gates only when a maximum age is configured
    old = verdict(tmp_path, True, time_unix=1000)
    assert daemon(["check"], {**env, "FABRIC_PROBE_VERDICT_PATH": old}).returncode == 0
    r = daemon(["check"], {**env, "FABRIC_PROBE_VERDICT_PATH": old, "FABRIC_PROBE_MAX_AGE_S": "60"})
    assert r.returncode == 1 and "stale" in r.stderr


def test_run_requires_cdi_env():
    r = daemon(["run", "--once"], {})
    assert r.returncode == 1
    assert "CDI container edits did not apply -- is CDI enabled in your container runtime?" in r.stderr  # main.go:218


def test_usage():
    assert daemon([]).returncode == 2


@pytest.mark.skipif(gpu_count() > 0, reason="CPU-only behaviour")
def test_run_without_gpu_does_not_gate(tmp_path):
    """No driver: the probe is 'not supported', no verdict is written and check() keeps passing —
    there is no CPU stand-in that would write a fake verdict."""
    v = tmp_path / "fabricprobe.json"
    r = daemon(["run", "--once"], {"COMPUTE_DOMAIN_UUID": "cd-1", "CDPROBE_LIBRARY": LIB,
                                   "FABRIC_PROBE_VERDICT_PATH": str(v)})
    assert r.returncode == 0 and "fabric probe not supported on this node" in r.stderr
    assert not v.exists()
    assert daemon(["check"], {"CLIQUE_ID": "", "FABRIC_PROBE_VERDICT_PATH": str(v)}).returncode == 0


@pytest.mark.gpu
def test_run_once_writes_a_passing_verdict_and_check_reads_it(tmp_path):
    v = tmp_path / "fabricprobe.json"
    # defaults on purpose (1 GiB per GPU, library gate): this is what the daemon pod would run
    m = tmp_path / "fabricprobe.prom"
    env = {"COMPUTE_DOMAIN_UUID": "cd-1", "CDPROBE_LIBRARY": LIB, "FABRIC_PROBE_VERDICT_PATH": str(v),
           "FABRIC_PROBE_METRICS_PATH": str(m)}
    r = daemon(["run", "--once"], env, timeout=300)
    assert r.returncode == 0, r.stderr
    assert "t_fabric_probe" in r.stderr and "fabric probe: verdict ok" in r.stderr
    d = json.loads(v.read_text())
    assert d["ok"] is True and d["unreachable_pairs"] == 0 and d["n"] == gpu_count() and d["probe_ms"] > 0
    n = d["n"]
    assert len(d["reach_read"]) == n * n and all(x == 1 for x in d["reach_read"]) and len(d["gbps_write"]) == n * n
    prom = m.read_text()
    assert "nvidia_dra_fabric_probe_duration_seconds" in prom and "nvidia_dra_fabric_probe_unreachable_pairs 0" in prom
    assert prom.count("nvidia_dra_fabric_probe_pair_gbps{") == 2 * (n * (n - 1) if n > 1 else 1)
    assert daemon(["check"], {"CLIQUE_ID": "", "FABRIC_PROBE_VERDICT_PATH": str(v)}).returncode == 0


# ---- round 2: one verdict schema for the Go patch and the C++ twin; stale verdicts; signals ------------
GO_DAEMON = os.path.join(ROOT, "integration", "cmd", "compute-domain-daemon", "fabricprobe.go")
GO_JSON_TYPE = {"int": int, "int64": int, "uint64": int, "bool": bool, "float32": (int, float), "float64": (int, float),
                "string": str, "[]int": (list, int), "[]float32": (list, (int, float))}


def go_verdict_schema():
    """{json key: python type} parsed from the struct tags of fabricProbeVerdict in the Go patch."""
    import re

    src = open(GO_DAEMON).read()
    body = src[src.index("type fabricProbeVerdict struct {"):]
    body = body[:body.index("\n}")]
    fields = re.findall(r"^\s*(\w+)\s+(\S+)\s+`json:\"(\w+)\"`", body, re.M)
    assert len(fields) >= 15
    return {tag: GO_JSON_TYPE[typ] for _, typ, tag in fields}


@pytest.mark.parametrize("ok", ["ok", "bad"])
def test_cpp_verdict_matches_the_go_struct_key_for_key(tmp_path, ok):
    """VERDICT r01 weak #5: the Go `check` must be able to read what the C++ `run` wrote and vice versa —
    same keys, same JSON types (reach cells are integers on both sides, min GB/s are carried)."""
    v = tmp_path / "fabricprobe.json"
    assert daemon(["selftest-verdict", str(v), ok], {"POD_UID": "pod-123"}).returncode == 0
    d = json.loads(v.read_text())
    schema = go_verdict_schema()
    assert set(d) == set(schema), (set(d) ^ set(schema))
    for key, typ in schema.items():
        if isinstance(typ, tuple) and typ[0] is list:
            assert isinstance(d[key], list) and all(isinstance(x, typ[1]) and not isinstance(x, bool) for x in d[key]), key
        else:
            assert isinstance(d[key], typ), key
            if typ is int:
                assert not isinstance(d[key], bool), key
    assert d["schema"] == 2 and d["pod_uid"] == "pod-123" and d["ok"] is (ok == "ok") and d["n"] == 2
    assert d["reach_write"] == ([1, 1, 1, 1] if ok == "ok" else [1, 0, 0, 1])
    assert d["min_gbps_read"] == pytest.approx(671.5) and d["gate_gbps_write"] == pytest.approx(625.7)
    # and the C++ check reads it back with the numbers in the message (they were always 0 in round 1's Go text)
    r = daemon(["check"], {"CLIQUE_ID": "", "FABRIC_PROBE_VERDICT_PATH": str(v), "POD_UID": "pod-123"})
    if ok == "ok":
        assert r.returncode == 0
    else:
        assert r.returncode == 1
        assert "fabric probe failed: 2 unreachable pair(s), 0 slow pair(s), min read 672 GB/s, min write 702 GB/s: synthetic" in r.stderr


def test_go_patch_is_internally_consistent():
    """The Go files cannot be compiled here; at least every identifier the daemon patch uses from the shim,
    the gate and the metrics package exists there with the name and arity it is called with."""
    import re

    d = open(GO_DAEMON).read()
    shim = open(os.path.join(ROOT, "integration", "pkg", "fabricprobe", "fabricprobe.go")).read()
    stub = open(os.path.join(ROOT, "integration", "pkg", "fabricprobe", "fabricprobe_stub.go")).read()
    gate = open(os.path.join(ROOT, "integration", "pkg", "featuregates", "fabricprobe_gate.go")).read()
    met = open(os.path.join(ROOT, "integration", "pkg", "metrics", "fabricprobe.go")).read()
    for name in set(re.findall(r"\bfabricprobe\.([A-Z]\w+)", re.sub(r"//.*", "", d))):
        assert re.search(rf"\b{name}\b", shim), f"pkg/fabricprobe lacks {name}"
        assert re.search(rf"\b{name}\b", stub), f"the !cgo stub lacks {name}"
    for fld in set(re.findall(r"\bres\.(\w+)", d)):
        assert re.search(rf"\b{fld}\b", shim[shim.index("type Result struct"):shim.index("type Probe struct")]), fld
        assert re.search(rf"\b{fld}\b", stub[stub.index("type Result struct"):stub.index("type Probe struct")]), fld
    for fld in set(re.findall(r"fabricprobe\.Config\{([^}]*)\}", d, re.S)[0].split()):
        if fld.endswith(":"):
            assert re.search(rf"\b{fld[:-1]}\b", shim[shim.index("type Config struct"):shim.index("type Result struct")]), fld
    assert "FabricProbe featuregate.Feature" in gate and "featuregates.FabricProbe" in d
    assert "func ObserveFabricProbe(node string, d time.Duration, ok bool, unreachable, slow, n int, gbpsRead, gbpsWrite []float32)" in met
    assert len(re.findall(r"metrics\.ObserveFabricProbe\(([^)]*)\)", d)[0].split(",")) == 8
    # the update channel keeps its single receiver (ADVICE r01): the patch never receives from it
    assert "GetDaemonInfoUpdateChan()" not in re.sub(r"//.*", "", d)
    # every C symbol the shim binds is one the header declares
    hdr = open(os.path.join(ROOT, "include", "cdprobe.h")).read()
    for sym in set(re.findall(r'dlsym\(cdp_dl, "(\w+)"\)', shim)):
        assert f" {sym}(" in hdr, sym
    for fld in set(re.findall(r"\br\.(\w+)", shim)) | set(re.findall(r"\bc\.(\w+) = ", shim)):
        assert re.search(rf"\b{fld}\b", hdr), f"cdprobe.h has no field {fld}"


def test_check_ignores_a_verdict_it_does_not_own(tmp_path):
    """ADVICE r01: /imexd outlives pods.  A failing verdict stamped by another pod, or from before a reboot,
    must not keep this pod NotReady (and a passing one must not make it Ready — it is simply not there)."""
    other = verdict(tmp_path, False, unreachable=3, pod_uid="pod-old", boot_id="")
    assert daemon(["check"], {"CLIQUE_ID": "", "FABRIC_PROBE_VERDICT_PATH": other, "POD_UID": "pod-new"}).returncode == 0
    assert daemon(["check"], {"CLIQUE_ID": "", "FABRIC_PROBE_VERDICT_PATH": other, "POD_UID": "pod-old"}).returncode == 1
    rebooted = verdict(tmp_path, False, unreachable=3, pod_uid="", boot_id="00000000-dead-beef-0000-000000000000")
    assert daemon(["check"], {"CLIQUE_ID": "", "FABRIC_PROBE_VERDICT_PATH": rebooted}).returncode == 0
    # periodic re-probe configured => a verdict must keep coming (default max age 3 x interval + 60 s)
    old = verdict(tmp_path, True, time_unix=1000)
    r = daemon(["check"], {"CLIQUE_ID": "", "FABRIC_PROBE_VERDICT_PATH": old, "FABRIC_PROBE_INTERVAL_S": "10"})
    assert r.returncode == 1 and "stale" in r.stderr


@pytest.mark.skipif(gpu_count() > 0, reason="CPU-only behaviour")
def test_run_removes_a_stale_verdict_at_startup(tmp_path):
    """A verdict left in the mount by a previous pod is gone once `run` has started, even when the probe turns
    out to be unsupported on this node (round 1 left a stale ok:false in place forever)."""
    v = tmp_path / "fabricprobe.json"
    v.write_text(json.dumps({"ok": False, "unreachable_pairs": 9, "time_unix": 5}))
    r = daemon(["run", "--once"], {"COMPUTE_DOMAIN_UUID": "cd-1", "CDPROBE_LIBRARY": LIB, "FABRIC_PROBE_VERDICT_PATH": str(v)})
    assert r.returncode == 0 and not v.exists()


@pytest.mark.gpu
def test_run_loop_reprobes_on_sigusr1_and_exits_on_sigterm(tmp_path):
    """The daemon loop itself: first pass at start, another on SIGUSR1 (the stand-in for a daemon-set update),
    SIGTERM ends it — signals are only deliverable inside the wait, so none is lost (ADVICE r01)."""
    import signal
    import time

    v = tmp_path / "fabricprobe.json"
    env = {"PATH": os.environ.get("PATH", ""), "LD_LIBRARY_PATH": os.environ.get("LD_LIBRARY_PATH", ""),
           "COMPUTE_DOMAIN_UUID": "cd-1", "CDPROBE_LIBRARY": LIB, "FABRIC_PROBE_VERDICT_PATH": str(v),
           "FABRIC_PROBE_BYTES": str(64 << 20), "POD_UID": "pod-7"}
    p = subprocess.Popen([DAEMON, "run"], env=env, stderr=subprocess.PIPE, text=True)
    try:
        t_end = time.time() + 240
        while not v.exists() and time.time() < t_end:
            time.sleep(0.1)
        first = json.loads(v.read_text())
        assert first["ok"] is True and first["pod_uid"] == "pod-7"
        for k in range(3):  # a burst: the second and third may coalesce, none may be lost for good
            p.send_signal(signal.SIGUSR1)
        time.sleep(2.0)
        p.send_signal(signal.SIGTERM)
        err = p.communicate(timeout=60)[1]
    finally:
        if p.poll() is None:
            p.kill()
    assert p.returncode == 0 and "Exiting" in err
    assert err.count("t_fabric_probe") >= 2


# ---- the daemon's run loop on a box WITHOUT a GPU: a test double of libcdprobe.so (tests/c/fake_cdprobe.c) ----------
@pytest.fixture(scope="module")
def fake_lib(tmp_path_factory):
    out = tmp_path_factory.mktemp("fake") / "libfake_cdprobe.so"
    subprocess.run(["gcc", "-shared", "-fPIC", "-O1", "-Wall", os.path.join(ROOT, "tests", "c", "fake_cdprobe.c"), "-o", str(out)],
                   check=True)
    return str(out)


def fake_env(tmp_path, fake_lib, script, **kw):
    e = {"PATH": os.environ.get("PATH", ""), "COMPUTE_DOMAIN_UUID": "cd-1", "CDPROBE_LIBRARY": fake_lib, "POD_UID": "pod-9",
         "FABRIC_PROBE_VERDICT_PATH": str(tmp_path / "fabricprobe.json"), "FAKE_CDPROBE_SCRIPT": script,
         "FAKE_CDPROBE_LOG": str(tmp_path / "calls.log"), "CDPROBE_NVML_PATH": "/nonexistent"}
    e.update(kw)
    return e


def calls(tmp_path):
    p = tmp_path / "calls.log"
    return p.read_text().split("\n")[:-1] if p.exists() else []


@pytest.mark.parametrize("script,ok,needle", [
    ("ok", True, "fabric probe: verdict ok, 2 GPU(s), 0 unreachable pair(s), 0 slow pair(s), min read 674 GB/s"),
    ("slow", False, "fabric probe: verdict FAILED, 2 GPU(s), 0 unreachable pair(s), 2 slow pair(s), min read 310 GB/s"),
    ("unreachable", False, "2 unreachable pair(s), 0 slow pair(s)"),
])
def test_run_once_through_the_real_writer(tmp_path, fake_lib, script, ok, needle):
    """`run --once` end to end on CPU: the verdict file the real run path writes matches the Go struct key for key,
    carries the pod uid, and `check` answers accordingly — a slow-but-reachable domain is NotReady with its own text."""
    env = fake_env(tmp_path, fake_lib, script)
    r = subprocess.run([DAEMON, "run", "--once"], env=env, capture_output=True, text=True, timeout=60)
    assert r.returncode == (0 if ok else 2) and needle in r.stderr, r.stderr
    d = json.loads((tmp_path / "fabricprobe.json").read_text())
    assert set(d) == set(go_verdict_schema()) and d["ok"] is ok and d["pod_uid"] == "pod-9" and d["n"] == 2
    assert d["slow_pairs"] == (2 if script == "slow" else 0) and d["gate_gbps_read"] == 604.0
    c = daemon(["check"], {"CLIQUE_ID": "", "FABRIC_PROBE_VERDICT_PATH": env["FABRIC_PROBE_VERDICT_PATH"], "POD_UID": "pod-9"})
    assert c.returncode == (0 if ok else 1)
    if script == "slow":
        assert "fabric probe failed: 0 unreachable pair(s), 2 slow pair(s), min read 310 GB/s, min write 705 GB/s" in c.stderr
    assert calls(tmp_path) == ["open 1", f"{script} 1", "close 1"]


def test_run_loop_reopens_after_a_timeout_and_reprobes_on_signal(tmp_path, fake_lib):
    """ADVICE r01: after a timed-out pass the handle may be sticky.  The loop writes a well-formed FAILING verdict
    for that pass, closes the handle, opens a fresh one for the next pass (SIGUSR1 = a daemon-set change), writes the
    passing verdict, and leaves on SIGTERM with every handle closed.  No signal is lost (sigsuspend-style wait)."""
    import signal
    import time

    env = fake_env(tmp_path, fake_lib, "timeout,ok")
    v = tmp_path / "fabricprobe.json"
    p = subprocess.Popen([DAEMON, "run"], env=env, stderr=subprocess.PIPE, text=True)
    try:
        t_end = time.time() + 30
        while not v.exists() and time.time() < t_end:
            time.sleep(0.02)
        first = json.loads(v.read_text())
        assert first["ok"] is False and "probe timed out" in first["error"] and "device watchdog fired" in first["error"]
        assert first["n"] == 2 and first["reach_read"] == [0, 0, 0, 0]  # the zeroed result of the failed pass, not garbage
        assert daemon(["check"], {"CLIQUE_ID": "", "FABRIC_PROBE_VERDICT_PATH": str(v), "POD_UID": "pod-9"}).returncode == 1
        time.sleep(0.2)  # let the loop reach its wait
        p.send_signal(signal.SIGUSR1)
        t_end = time.time() + 30
        while time.time() < t_end and not json.loads(v.read_text())["ok"]:
            time.sleep(0.02)
        assert json.loads(v.read_text())["ok"] is True
        assert daemon(["check"], {"CLIQUE_ID": "", "FABRIC_PROBE_VERDICT_PATH": str(v), "POD_UID": "pod-9"}).returncode == 0
        p.send_signal(signal.SIGTERM)
        err = p.communicate(timeout=30)[1]
    finally:
        if p.poll() is None:
            p.kill()
    assert p.returncode == 0 and "Exiting" in err and err.count("t_fabric_probe") == 2
    assert calls(tmp_path) == ["open 1", "timeout 1", "close 1", "open 2", "ok 2", "close 2"]


def test_run_loop_periodic_passes_and_burst_of_signals(tmp_path, fake_lib):
    """FABRIC_PROBE_INTERVAL_S: a pass every second without any signal; a burst of SIGUSR1 coalesces but is never lost."""
    import signal
    import time

    env = fake_env(tmp_path, fake_lib, "ok", FABRIC_PROBE_INTERVAL_S="1")
    p = subprocess.Popen([DAEMON, "run"], env=env, stderr=subprocess.PIPE, text=True)
    try:
        time.sleep(2.6)
        n_periodic = len([c for c in calls(tmp_path) if c.startswith("ok")])
        assert 2 <= n_periodic <= 4
        for _ in range(5):
            p.send_signal(signal.SIGUSR1)
        time.sleep(0.5)
        assert len([c for c in calls(tmp_path) if c.startswith("ok")]) >= n_periodic + 1
        p.send_signal(signal.SIGTERM)
        err = p.communicate(timeout=30)[1]
    finally:
        if p.poll() is None:
            p.kill()
    assert p.returncode == 0 and "Exiting" in err
    assert calls(tmp_path)[0] == "open 1" and calls(tmp_path)[-1] == "close 1"  # one handle for the whole life: no pass failed


def test_open_failure_is_not_ready_but_unsupported_does_not_gate(tmp_path, fake_lib):
    env = fake_env(tmp_path, fake_lib, "openfail,ok")
    v = tmp_path / "fabricprobe.json"
    v.write_text(json.dumps({"ok": True, "time_unix": 5}))  # a stale ok:true from a previous pod must not survive
    r = subprocess.run([DAEMON, "run", "--once"], env=env, capture_output=True, text=True, timeout=60)
    assert r.returncode == 1 and "error opening fabric probe: CUDA call failed: fake: cuMemCreate" in r.stderr
    d = json.loads(v.read_text())
    assert d["ok"] is False and "cdprobe_open: CUDA call failed" in d["error"] and d["pod_uid"] == "pod-9"
    assert daemon(["check"], {"CLIQUE_ID": "", "FABRIC_PROBE_VERDICT_PATH": str(v), "POD_UID": "pod-9"}).returncode == 1
    # unsupported (no sm_90 GPU): no verdict at all, check does not gate — and the stale file is gone too
    v.write_text(json.dumps({"ok": False, "time_unix": 5, "unreachable_pairs": 3}))
    r = subprocess.run([DAEMON, "run", "--once"], env=fake_env(tmp_path, fake_lib, "unsupported"), capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and "fabric probe not supported on this node" in r.stderr and not v.exists()
    assert daemon(["check"], {"CLIQUE_ID": "", "FABRIC_PROBE_VERDICT_PATH": str(v)}).returncode == 0


# ---- the closest thing to `go vet` without a Go toolchain: lexical checks that catch whole classes of compile errors ----
GO_FILES = [os.path.join(ROOT, "integration", *p) for p in (
    ("cmd", "compute-domain-daemon", "fabricprobe.go"), ("pkg", "fabricprobe", "fabricprobe.go"),
    ("pkg", "fabricprobe", "fabricprobe_stub.go"), ("pkg", "featuregates", "fabricprobe_gate.go"),
    ("pkg", "metrics", "fabricprobe.go"), ("internal", "common", "topology.go"))]


def _go_strip(src):
    """Go source with comments, strings, runes and the cgo preamble blanked out (lengths preserved)."""
    out, i, n = [], 0, len(src)
    while i < n:
        c = src[i]
        two = src[i:i + 2]
        if two == "//":
            j = src.find("\n", i)
            j = n if j < 0 else j
            out.append(" " * (j - i))
            i = j
        elif two == "/*":
            j = src.find("*/", i + 2)
            j = n if j < 0 else j + 2
            out.append("".join("\n" if ch == "\n" else " " for ch in src[i:j]))
            i = j
        elif c in "\"`'":
            j = i + 1
            while j < n and src[j] != c:
                j += 2 if (src[j] == "\\" and c != "`") else 1
            out.append(c + "".join("\n" if ch == "\n" else " " for ch in src[i + 1:j]) + c)
            i = j + 1
        else:
            out.append(c)
            i += 1
    return "".join(out)


@pytest.mark.parametrize("path", GO_FILES, ids=[os.path.relpath(p, ROOT) for p in GO_FILES])
def test_go_file_is_lexically_sound(path):
    """Balanced brackets, a package clause, and — Go rejects both — no import that is never used and no package
    qualifier that was never imported."""
    import re

    src = open(path).read()
    code = _go_strip(src)
    stack = []
    pairs = {")": "(", "]": "[", "}": "{"}
    for k, ch in enumerate(code):
        if ch in "([{":
            stack.append((ch, k))
        elif ch in ")]}":
            assert stack and stack[-1][0] == pairs[ch], f"unbalanced {ch!r} at line {code[:k].count(chr(10)) + 1}"
            stack.pop()
    assert not stack, f"unclosed {stack[-1][0]!r} opened at line {code[:stack[-1][1]].count(chr(10)) + 1}"
    assert re.search(r"^package \w+$", code, re.M)
    # imports: (alias, path) pairs from the original source (paths are strings, blanked in `code`)
    imports = []
    for block in re.findall(r"^import \((.*?)^\)", src, re.M | re.S):
        imports += re.findall(r"^\s*(?:(\w+)\s+)?\"([^\"]+)\"", block, re.M)
    imports += [(a, p) for a, p in re.findall(r"^import (?:(\w+)\s+)?\"([^\"]+)\"", src, re.M)]
    assert imports or "import" not in code
    special = {"k8s.io/klog/v2": "klog", "github.com/urfave/cli/v2": "cli"}
    names = {}
    for alias, ipath in imports:
        names[alias or special.get(ipath, ipath.rsplit("/", 1)[-1])] = ipath
    body = code[code.index("\n", max(code.rfind("import ("), 0)):]
    for name, ipath in names.items():
        assert re.search(rf"\b{re.escape(name)}\.", body), f"{ipath} imported and not used"
    # every lower-case package qualifier in use is imported (catches a forgotten import)
    known = set(names) | {"C"}
    used = set(re.findall(r"(?<![\w.)\]])([a-z][a-z0-9]*)\.[A-Z]\w*", body))
    locals_ = set(re.findall(r"\b([a-z]\w*)\s*(?::=|,|\))", body)) | set(re.findall(r"\b([a-z]\w*) \*?[\w.\[\]]+[,)]", body))
    for q in used - known - locals_:
        # receivers, struct values and parameters (v.OK, res.N, flags.podUID, cfg.Bytes ...) are not packages
        assert re.search(rf"\b(?:var\s+{q}\b|{q}\s*:?=|func\s*\(\s*{q}\s|\b{q}\s+[\w.*\[\]]+\s*[,)]|\b{q},)", body), f"{q}. used but never imported or declared"
