"""cdprobe_diagnose without a GPU: the ABI layout, the word classifier of probe_types.h against words the CPU oracle
generates, the daemon's diagnosis log line (through a test double of the library), and the Go mirror."""
import ctypes as C
import json
import os
import re
import subprocess

import pytest

from conftest import ROOT
from harness import assert_layout, c_tool, exported_symbols, header_values

HEADER = os.path.join(ROOT, "include", "cdprobe.h")
CSRC = os.path.join(ROOT, "k8s-dra-driver-gpu_b200", "csrc")
DAEMON = os.path.join(ROOT, "k8s-dra-driver-gpu_b200", "cdprobe-daemon")
SEED = 0xCD5EED0000000001
FLIP, ZERO, DISPLACED, STALE, FOREIGN = 0, 1, 2, 3, 4


def test_diag_struct_layout_matches_c(pkg, tmp_path):
    a = pkg.abi
    structs = {"cdprobe_diag_sample_t": a.DiagSampleT, "cdprobe_diag_t": a.DiagT}
    assert_layout(tmp_path, structs)
    samples, *kinds = header_values(tmp_path, "CDPROBE_DIAG_SAMPLES", "CDPROBE_DIAG_FLIP", "CDPROBE_DIAG_ZERO",
                                    "CDPROBE_DIAG_DISPLACED", "CDPROBE_DIAG_STALE", "CDPROBE_DIAG_FOREIGN")
    assert samples == a.DIAG_SAMPLES
    assert kinds == [a.DIAG_FLIP, a.DIAG_ZERO, a.DIAG_DISPLACED, a.DIAG_STALE, a.DIAG_FOREIGN]
    assert "cdprobe_diagnose" in a.SYMBOLS


# ---- the classifier: known answers built with the oracle's forward functions ------------------------------------
@pytest.fixture(scope="module")
def classify(tmp_path_factory):
    run = c_tool(tmp_path_factory, "diag_classify.cc", "-O1")
    return lambda cases: [tuple(r) for r in run(cases)]


def test_read_cell_words_classify_to_their_rank_and_index(oracle, classify):
    L = oracle.lib()
    n_ranks, target, words = 16, 5, 4096
    src_words, first = 15 * words, 2 * words  # sliced, 16 ranks: 15 slices; the cell reads slice 2
    spec = ("read", SEED, n_ranks, target, first, words, src_words)
    cases, want = [], []
    for r in (0, target, 15):
        for kp in (0, words - 1, first + 7, src_words - 1):
            cases.append((*spec, 7, L.cdoracle_src_word(SEED, r, kp)))
            want.append((DISPLACED if r == target else FOREIGN, r, kp, 0))
    for r, kp in ((target, src_words), (3, src_words), (16, 5)):  # one past the end; a rank outside the domain
        cases.append((*spec, 7, L.cdoracle_src_word(SEED, r, kp)))
        want.append((FLIP, -1, 0, 0))
    cases.append((*spec, 7, 0))
    want.append((ZERO, -1, 0, 0))
    for k, mask in ((0, 1), (7, 1 << 63), (words - 1, 0xFF00), (100, 0x0123456789ABCDEF)):
        cases.append((*spec, k, L.cdoracle_src_word(SEED, target, first + k) ^ mask))
        want.append((FLIP, -1, 0, 0))
    # rank 15 is FOREIGN only in a domain that has a rank 15
    cases.append(("read", SEED, 4, 1, 0, words, 3 * words, 0, L.cdoracle_src_word(SEED, 15, 9)))
    want.append((FLIP, -1, 0, 0))
    got = classify(cases)
    for c, g, w in zip(cases, got, want):
        assert g[0] == L.cdoracle_src_word(SEED, c[3], c[4] + c[7]), c  # the expected word is the oracle's
        assert g[1:] == w, (c, g, w)


def test_write_cell_words_classify_to_their_writer_and_run(oracle, classify):
    L = oracle.lib()
    n_ranks, issuer, target, run_seq, words = 16, 3, 9, 20, 4096
    spec = ("write", SEED, n_ranks, issuer, target, run_seq, words)

    def ww(src, seq, k):
        return L.cdoracle_write_word(L.cdoracle_write_salt(SEED, src, target, seq), k)

    cases, want = [], []
    for kp in (0, 1, words - 1):
        cases.append((*spec, 5, ww(issuer, run_seq, kp)))
        want.append((DISPLACED, issuer, kp, 0))
        for d in range(1, 9):
            cases.append((*spec, 5, ww(issuer, run_seq - d, kp)))
            want.append((STALE, issuer, kp, run_seq - d))
        cases.append((*spec, 5, ww(issuer, run_seq - 9, kp)))  # older than 8 runs: not traced back
        want.append((FLIP, -1, 0, 0))
        for r in (0, 1, 8, target, 15):
            cases.append((*spec, 5, ww(r, run_seq, kp)))
            want.append((FOREIGN, r, kp, 0))
    for src, seq in ((issuer, run_seq), (issuer, run_seq - 1), (15, run_seq)):  # one past the slot
        cases.append((*spec, 5, ww(src, seq, words)))
        want.append((FLIP, -1, 0, 0))
    cases.append((*spec, 5, ww(issuer, run_seq, words + 10 ** 9)))
    want.append((FLIP, -1, 0, 0))
    cases.append((*spec, 5, 0))
    want.append((ZERO, -1, 0, 0))
    for k, mask in ((0, 1 << 17), (5, 0xFF00), (words - 1, 1 << 63)):
        cases.append((*spec, k, ww(issuer, run_seq, k) ^ mask))
        want.append((FLIP, -1, 0, 0))
    # early runs: no candidate before run 1
    early = ("write", SEED, 2, 0, 1, 3, words)
    cases += [(*early, 0, L.cdoracle_write_word(L.cdoracle_write_salt(SEED, 0, 1, 1), 4)),
              (*early, 0, L.cdoracle_write_word(L.cdoracle_write_salt(SEED, 0, 1, 0), 4))]
    want += [(STALE, 0, 4, 1), (FLIP, -1, 0, 0)]
    got = classify(cases)
    for c, g, w in zip(cases, got, want):
        assert g[0] == L.cdoracle_write_word(L.cdoracle_write_salt(SEED, c[3], c[4], c[5]), c[7]), c
        assert g[1:] == w, (c, g, w)


# ---- the daemon's log line, through a test double of libcdprobe.so ----------------------------------------------
@pytest.fixture(scope="module")
def fake_libs(pkg, tmp_path_factory):
    d = tmp_path_factory.mktemp("fakediag")
    src = os.path.join(ROOT, "tests", "c", "fake_cdprobe_diagnose.c")
    with_sym, without = str(d / "libfake_diag.so"), str(d / "libfake_nodiag.so")
    subprocess.run(["gcc", "-shared", "-fPIC", "-O1", "-Wall", src, "-o", with_sym], check=True)
    subprocess.run(["gcc", "-shared", "-fPIC", "-O1", "-Wall", "-DFAKE_CDPROBE_NO_DIAGNOSE", src, "-o", without], check=True)
    assert "cdprobe_diagnose" in exported_symbols(with_sym)
    assert "cdprobe_diagnose" not in exported_symbols(without)
    return with_sym, without


def run_once(tmp_path, lib, script):
    env = {"PATH": os.environ.get("PATH", ""), "COMPUTE_DOMAIN_UUID": "cd-1", "CDPROBE_LIBRARY": lib, "POD_UID": "pod-9",
           "FABRIC_PROBE_VERDICT_PATH": str(tmp_path / "fabricprobe.json"), "FAKE_CDPROBE_SCRIPT": script,
           "FAKE_CDPROBE_LOG": str(tmp_path / "calls.log"), "CDPROBE_NVML_PATH": "/nonexistent"}
    r = subprocess.run([DAEMON, "run", "--once"], env=env, capture_output=True, text=True, timeout=60)
    log = tmp_path / "calls.log"
    return r, json.loads((tmp_path / "fabricprobe.json").read_text()), log.read_text().split("\n")[:-1]


def verdict_keys(tmp_path):
    v = tmp_path / "selftest.json"
    assert subprocess.run([DAEMON, "selftest-verdict", str(v), "bad"], capture_output=True).returncode == 0
    return set(json.loads(v.read_text()))


def test_daemon_logs_where_an_integrity_failure_happened(tmp_path, fake_libs):
    r, v, calls = run_once(tmp_path, fake_libs[0], "corrupt")
    assert r.returncode == 2, r.stderr
    lines = [l for l in r.stderr.splitlines() if l.startswith("fabric probe diagnosis:")]
    assert lines == ["fabric probe diagnosis: read 1 -> 0, reader 1: 3/134217728 bad words, 2 bad granule(s), first bad "
                     "byte 4104; flip 3 zero 0 displaced 0 stale 0 foreign 0; bits 17:2 8:1; in transit"]
    # the issuer's read, then the target's: nothing else is diagnosed
    assert calls == ["open 1", "corrupt 1", "diagnose 1101", "diagnose 1100", "close 1"]
    assert set(v) == verdict_keys(tmp_path) and v["ok"] is False and v["unreachable_pairs"] == 1


def test_daemon_diagnoses_nothing_on_a_healthy_pass(tmp_path, fake_libs):
    r, v, calls = run_once(tmp_path, fake_libs[0], "ok")
    assert r.returncode == 0 and "diagnosis" not in r.stderr and v["ok"] is True
    assert calls == ["open 1", "ok 1", "close 1"]


def test_daemon_runs_with_a_library_without_diagnose(tmp_path, fake_libs):
    r, v, calls = run_once(tmp_path, fake_libs[1], "corrupt")
    assert r.returncode == 2 and "fabric probe: verdict FAILED, 2 GPU(s), 1 unreachable pair(s)" in r.stderr
    assert "diagnosis" not in r.stderr
    assert calls == ["open 1", "corrupt 1", "close 1"]
    assert set(v) == verdict_keys(tmp_path)


# ---- Go mirror ----------------------------------------------------------------------------------------------------
def test_go_diagnose_is_consistent_across_shim_stub_and_daemon():
    go = os.path.join(ROOT, "integration")
    d = re.sub(r"//.*", "", open(os.path.join(go, "cmd", "compute-domain-daemon", "fabricprobe.go")).read())
    shim = open(os.path.join(go, "pkg", "fabricprobe", "fabricprobe.go")).read()
    stub = open(os.path.join(go, "pkg", "fabricprobe", "fabricprobe_stub.go")).read()

    def struct(src, name):
        body = src[src.index(f"type {name} struct {{"):]
        return body[:body.index("\n}")]

    used = set(re.findall(r"\b(?:diag|at)\.([A-Z]\w*)", d))
    assert {"BadWords", "Words", "BadGranules", "FirstBad", "LastBad", "KindCount", "BitFlips"} <= used
    for src in (shim, stub):
        for fld in used:
            assert re.search(rf"\b{fld}\b", struct(src, "Diagnosis")), fld
        assert re.search(r"\bKind\b", struct(src, "DiagSample")) and "DiagKinds" in src
    assert "func (p *Probe) Diagnose(op uint32, issuer, target, reader int) (Diagnosis, error)" in shim
    assert "func (*Probe) Diagnose(uint32, int, int, int) (Diagnosis, error)" in stub
    assert "probe.Diagnose(" in d and "fabricprobe.ErrUnsupported" in d
    # optional binding: a missing symbol does not fail cdp_load
    assert 'dlsym(cdp_dl, "cdprobe_diagnose")' in shim
    required = re.search(r"if \(!cdp_open[^)]*\)", shim).group(0)
    assert "cdp_diag" not in required
    # the C shim reads only fields the header declares
    hdr = open(HEADER).read()
    for fld in set(re.findall(r"\bd\.(\w+)", shim)) | set(re.findall(r"\bs\.(\w+)\)", shim)):
        assert re.search(rf"\b{fld}\b", hdr), fld
    # the log line is the C++ twin's
    cpp = open(os.path.join(CSRC, "daemon_main.cc")).read()
    for piece in ("fabric probe diagnosis: %s %", "bad words, %", "bad granule(s), first bad byte %s; ",
                  "flip %", " zero %", " displaced %", " stale %", " foreign %", "; bits%s%s", "; in transit", "; at rest"):
        assert piece in cpp and piece in d, piece


def test_diagnose_rejects_a_null_handle(pkg):
    a = pkg.abi
    lib = a.load_library()
    d = a.DiagT()
    assert lib.cdprobe_diagnose(None, a.OP_READ, 0, 0, 0, C.byref(d)) == a.ERR_ARG
    assert lib.cdprobe_diagnose(None, a.OP_READ, 0, 0, 0, None) == a.ERR_ARG
