"""cdprobe_links without a GPU: its ABI, the payload rule of schedule.cc against links_ref, the NVML sampler of links.cc
against the fake libnvidia-ml.so.1 (tests/fake_nvml/fake_nvml_links.c), and what the C++ daemon logs and exports from it (DESIGN §5o).

links.cc and schedule.cc are compiled for the host next to small drivers, as test_large_regions_cpu.py does with
plan.cc; the daemon runs against the library test doubles tests/c/fake_cdprobe_links.c and, for a library without
cdprobe_links, tests/c/fake_cdprobe.c."""
import ctypes as C
import json
import os
import re
import subprocess
import textwrap

import pytest

import links_ref
from conftest import ROOT
from harness import assert_layout
from kernel_tools import CSRC

FAKE_NVML_DIR = os.path.join(ROOT, "tests", "fake_nvml")
HEADER = os.path.join(ROOT, "include", "cdprobe.h")
NVML_INC = "/usr/local/cuda/include"
GIB = 1 << 30
MODE_REACH_ONLY, MODE_SLICED, MODE_FULL = 0, 1, 2
LOCAL_DIAG, OVERLAP_VERIFY, UNIDIRECTIONAL = 0x04, 0x20, 0x80
TX, RX, REPLAY, RECOVERY, CRC = 138, 139, 161, 162, 163
NOT_SUPPORTED, UNKNOWN = 3, 999


def build_fake_nvml(d):
    """The fake libnvidia-ml.so.1 with the per-link counter entry points (tests/fake_nvml/fake_nvml_links.c), built in
    directory d; returns its path."""
    out = os.path.join(str(d), "libnvidia-ml.so.1")
    subprocess.run(["gcc", "-O1", "-fPIC", "-shared", "-Wall", "-I", NVML_INC, "-I", FAKE_NVML_DIR,
                    os.path.join(FAKE_NVML_DIR, "fake_nvml_links.c"), "-o", out], check=True)
    return out


def fake_uuid(g):
    return f"GPU-{0xb2000000 + g:08x}-fa4e-0000-0000-{g:012x}"


# ---- ABI --------------------------------------------------------------------------------------------------------
def test_layout_matches_gcc_offsetof(pkg, tmp_path):
    abi = pkg.abi
    assert_layout(tmp_path, {"cdprobe_links_t": abi.LinksT, "cdprobe_link_device_t": abi.LinkDeviceT})


def test_option_number_and_symbol(pkg):
    text = open(HEADER).read()
    assert re.search(r"#define CDPROBE_OPT_LINK_COUNTERS 27u", text)
    assert pkg.abi.OPT_LINK_COUNTERS == 27
    assert "CDPROBE_API int cdprobe_links(cdprobe_t* h, cdprobe_links_t* out);" in text
    assert pkg.abi.SYMBOLS["cdprobe_links"][1][1] is not None
    lib = pkg.abi.load_library()
    assert lib.cdprobe_links(None, None) == pkg.abi.ERR_ARG
    t = pkg.abi.LinksT()
    assert lib.cdprobe_links(None, C.byref(t)) == pkg.abi.ERR_ARG


def test_links_from_c(pkg):
    abi, fp = pkg.abi, pkg.fabricprobe
    t = abi.LinksT()
    t.abi, t.n_devices, t.run_seq, t.sample_ms = abi.ABI_VERSION, 2, 7, 0.25
    d = t.dev[1]
    d.status, d.rank_mask, d.uuid = 0, 0b1100, b"GPU-1"
    d.link_mask, d.lost_mask, d.error_mask = 0x3ffff, 1 << 11, 1 << 7
    d.expected_tx_kib, d.expected_rx_kib = 1024, 2048
    d.tx_kib[3], d.rx_kib[4] = 5, 6
    d.errors[7][abi.LINK_REPLAY], d.errors[7][abi.LINK_CRC] = 312, 41
    d.failed_fields[9] = abi.LINK_FIELD_RECOVERY
    d.remote_bus_id[7].value = b"0000:05:00.0"
    t.dev[2].uuid = b"beyond n_devices"
    L = fp.Links.from_c(t)
    assert (L.n_devices, L.run_seq, L.sample_ms, len(L.devices)) == (2, 7, 0.25, 2)
    x = L.devices[1]
    assert x["uuid"] == "GPU-1" and x["rank_mask"] == 0b1100 and x["lost_mask"] == 1 << 11
    assert x["tx_kib"][3] == 5 and x["rx_kib"][4] == 6 and len(x["tx_kib"]) == 18
    assert x["errors"][7] == {"replay": 312, "recovery": 0, "crc": 41}
    assert x["failed_fields"][9] == abi.LINK_FIELD_RECOVERY
    assert x["remote_bus_id"][7] == "0000:05:00.0" and x["remote_bus_id"][6] == ""
    assert (x["expected_tx_kib"], x["expected_rx_kib"]) == (1024, 2048)


def test_go_mirror_has_every_field(pkg):
    """The Go binding converts every field of cdprobe_link_device_t and cdprobe_links_t, binds cdprobe_links as an
    optional symbol, and the stub and the daemon carry the new flag and series."""
    shim = open(os.path.join(ROOT, "integration", "pkg", "fabricprobe", "fabricprobe.go")).read()
    stub = open(os.path.join(ROOT, "integration", "pkg", "fabricprobe", "fabricprobe_stub.go")).read()
    daemon = open(os.path.join(ROOT, "integration", "cmd", "compute-domain-daemon", "fabricprobe.go")).read()
    met = open(os.path.join(ROOT, "integration", "pkg", "metrics", "fabricprobe.go")).read()
    abi = pkg.abi
    for fname, _ in abi.LinkDeviceT._fields_:
        if fname != "reserved":
            assert f"d.{fname}" in shim, fname
    for fname in ("n_devices", "run_seq", "sample_ms"):
        assert f"t.{fname}" in shim, fname
    assert 'dlsym(cdp_dl, "cdprobe_links")' in shim
    assert "func (p *Probe) Links() (Links, error)" in shim and "func (p *Probe) Links() (Links, error)" in stub
    assert "OptLinkCounters = 27" in shim and "OptLinkCounters = 27" in stub
    assert '"fabric-probe-link-counters"' in daemon and "FABRIC_PROBE_LINK_COUNTERS" in daemon
    assert '"fabric_probe_link_kib"' in met and '"fabric_probe_link_errors"' in met


# ---- the payload rule ---------------------------------------------------------------------------------------------
PAYLOAD_MAIN = r"""
#include <stdio.h>
#include <string.h>
#include "plan.h"
#include "schedule.h"
// stdin, one case per line: n bytes mode ops flags warm ran_mask down_i down_j dev[0..n)
// stdout: rc then tx[0..n) rx[0..n) per device id
int main() {
  unsigned n, mode, ops, flags, ran; unsigned long long bytes, warm; int di, dj;
  while (scanf("%u %llu %u %u %u %llu %u %d %d", &n, &bytes, &mode, &ops, &flags, &warm, &ran, &di, &dj) == 9) {
    uint32_t dev[cdp::kMaxRanks];
    for (unsigned r = 0; r < n; ++r) scanf("%u", &dev[r]);
    cdp::Plan pl;
    int rc = cdp::make_plan(n, bytes, mode, flags, &pl);
    int32_t st[cdp::kMaxRanks][cdp::kMaxRanks];
    memset(st, 0, sizeof(st));
    if (di >= 0) st[di][dj] = CDPROBE_ERR_STATE;
    cdp::ScheduleInput in;
    in.plan = &pl; in.ops = ops; in.flags = flags; in.ctas = 132; in.verify_ctas = 32; in.status = st;
    uint64_t tx[cdp::kMaxRanks] = {}, rx[cdp::kMaxRanks] = {};
    if (rc == 0) cdp::link_payload(in, ran, dev, warm, tx, rx);
    printf("%d", rc);
    for (unsigned d = 0; d < n; ++d) printf(" %llu", (unsigned long long)tx[d]);
    for (unsigned d = 0; d < n; ++d) printf(" %llu", (unsigned long long)rx[d]);
    printf("\n");
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def host_payload(tmp_path_factory):
    d = tmp_path_factory.mktemp("payload")
    (d / "main.cc").write_text(PAYLOAD_MAIN)
    exe = d / "payload"
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", CSRC, str(d / "main.cc"), f"{CSRC}/plan.cc",
                    f"{CSRC}/schedule.cc", "-o", str(exe)], check=True)

    def run(cases):
        inp = "".join(" ".join(str(v) for v in (*c[:9], *c[9])) + "\n" for c in cases)
        out = subprocess.run([str(exe)], input=inp, capture_output=True, text=True, check=True).stdout.splitlines()
        res = []
        for (n, *_), line in zip(cases, out):
            v = [int(x) for x in line.split()]
            res.append((v[0], v[1:1 + n], v[1 + n:1 + 2 * n]))
        return res
    return run


def assignments(n):
    """Device of each rank: all on one device, all distinct, pairs sharing one, and two halves (two processes of
    n / 2 ranks, each process's ranks on one device)."""
    out = [[0] * n, list(range(n)), [r // 2 for r in range(n)]]
    if n >= 2:
        out.append([0 if r < n // 2 else 1 for r in range(n)])
    return out


def schedulable(pkg, n, mode, ops, flags):
    s = pkg.abi.ScheduleT()
    return pkg.abi.load_library().cdprobe_schedule(n, 0, GIB, mode, ops, flags, 132, 32, C.byref(s)) == 0


@pytest.mark.parametrize("n", range(1, 17))
def test_payload_equals_the_reference(pkg, host_payload, n):
    cases, want = [], []
    for mode in (MODE_REACH_ONLY, MODE_SLICED, MODE_FULL):
        pl = pkg.fabricprobe.plan(n, GIB, mode, 0)
        partner = [[pl.partner[r][g] for g in range(16)] for r in range(16)]
        for ops in (1, 2, 3):
            for flags in (OVERLAP_VERIFY, OVERLAP_VERIFY | LOCAL_DIAG, OVERLAP_VERIFY | UNIDIRECTIONAL, 0):
                if not schedulable(pkg, n, mode, ops, flags | (0 if flags else 0x100)):
                    continue
                for warm in (0, 8 << 20):
                    downs = [None] + ([(0, n - 1)] if n >= 2 else [])
                    for down in downs:
                        for dev in assignments(n):
                            ran = (1 << n) - 1
                            cases.append((n, GIB, mode, ops, flags, warm, ran, *(down or (-1, -1)), dev))
                            want.append(links_ref.payload(partner, pl.rounds, n, pl.bytes_per_pair, ops, dev, warm,
                                                          down=[down] if down else ()))
    got = host_payload(cases)
    assert len(got) == len(cases)
    for c, (rc, tx, rx), (wtx, wrx) in zip(cases, got, want):
        assert rc == 0, c
        assert tx == [wtx.get(d, 0) for d in range(n)], c
        assert rx == [wrx.get(d, 0) for d in range(n)], c
        if len(set(c[9])) == 1:
            assert not any(tx) and not any(rx), c  # every rank on one device: nothing leaves it


def test_payload_of_a_pair_by_hand(pkg, host_payload):
    """Two ranks on two devices, 1 GiB sliced: bytes_per_pair 1 GiB.  Reads only: each device sends its slice once and
    receives the peer's; a warm-up adds 8 MiB each way.  Writes only: the same, issued by the other side.  A rank that
    did not run adds nothing of its own jobs."""
    bpp = GIB
    rc, tx, rx = host_payload([(2, GIB, MODE_SLICED, 1, OVERLAP_VERIFY, 8 << 20, 3, -1, -1, [0, 1])])[0]
    assert rc == 0 and tx == [bpp + (8 << 20)] * 2 and rx == tx
    rc, tx, rx = host_payload([(2, GIB, MODE_SLICED, 1, OVERLAP_VERIFY, 0, 1, -1, -1, [0, 1])])[0]
    assert (tx, rx) == ([0, bpp], [bpp, 0])  # rank 0 read rank 1's slice: rank 1's device sent it
    rc, tx, rx = host_payload([(2, GIB, MODE_SLICED, 2, OVERLAP_VERIFY, 0, 1, -1, -1, [0, 1])])[0]
    assert (tx, rx) == ([bpp, 0], [0, bpp])  # rank 0 wrote into rank 1
    rc, tx, rx = host_payload([(2, GIB, MODE_SLICED, 3, OVERLAP_VERIFY, 0, 3, 0, 1, [0, 1])])[0]
    assert (tx, rx) == ([0, 0], [0, 0])  # the pair's only cell is down


# ---- the sampler against the fake NVML ---------------------------------------------------------------------------
SAMPLER_MAIN = r"""
#include <stdio.h>
#include <string.h>
#include "links.h"
// argv: uuids (a leading "MIG:" marks a MIG instance).  Samples every device twice and prints one JSON row each.
int main(int argc, char** argv) {
  static char uuid[CDPROBE_MAX_GPUS][48];
  bool mig[CDPROBE_MAX_GPUS] = {};
  uint32_t n = (uint32_t)(argc - 1);
  for (uint32_t d = 0; d < n; ++d) {
    const char* u = argv[d + 1];
    if (!strncmp(u, "MIG:", 4)) { mig[d] = true; u += 4; }
    snprintf(uuid[d], 48, "%s", u);
  }
  static cdp::LinkSampler s;
  static cdp::LinkSample a[CDPROBE_MAX_GPUS], b[CDPROBE_MAX_GPUS];
  s.open(n, uuid, mig);
  s.sample(a, true);
  s.sample(b, false);
  for (uint32_t d = 0; d < n; ++d) {
    cdprobe_link_device_t row;
    memset(&row, 0, sizeof(row));
    cdp::link_delta(a[d], b[d], &row);
    printf("{\"status\": %d, \"link_mask\": %u, \"lost_mask\": %u, \"error_mask\": %u, \"tx_kib\": [", row.status,
           row.link_mask, row.lost_mask, row.error_mask);
    for (int l = 0; l < 18; ++l) printf("%s%llu", l ? ", " : "", (unsigned long long)row.tx_kib[l]);
    printf("], \"rx_kib\": [");
    for (int l = 0; l < 18; ++l) printf("%s%llu", l ? ", " : "", (unsigned long long)row.rx_kib[l]);
    printf("], \"errors\": [");
    for (int l = 0; l < 18; ++l)
      printf("%s[%llu, %llu, %llu]", l ? ", " : "", (unsigned long long)row.errors[l][0],
             (unsigned long long)row.errors[l][1], (unsigned long long)row.errors[l][2]);
    printf("], \"failed_fields\": [");
    for (int l = 0; l < 18; ++l) printf("%s%u", l ? ", " : "", row.failed_fields[l]);
    printf("], \"remote_bus_id\": [");
    for (int l = 0; l < 18; ++l) printf("%s\"%s\"", l ? ", " : "", row.remote_bus_id[l]);
    printf("]}\n");
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def sampler(tmp_path_factory):
    d = tmp_path_factory.mktemp("sampler")
    fake_nvml = build_fake_nvml(d)
    (d / "main.cc").write_text(SAMPLER_MAIN)
    exe = d / "sampler"
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", CSRC, "-I", NVML_INC, str(d / "main.cc"),
                    f"{CSRC}/links.cc", "-o", str(exe), "-ldl"], check=True)

    def run(tmp_path, scenario, uuids, nvml=fake_nvml):
        sc = tmp_path / "scenario.txt"
        sc.write_text(textwrap.dedent(scenario))
        env = dict(os.environ, FAKE_NVML_SCENARIO=str(sc), CDPROBE_NVML_PATH=nvml)
        out = subprocess.run([str(exe), *uuids], env=env, capture_output=True, text=True, timeout=60, check=True)
        return [json.loads(l) for l in out.stdout.splitlines()]
    return run


def clean(link_mask=(1 << 18) - 1):
    return {"status": 0, "link_mask": link_mask, "lost_mask": 0, "error_mask": 0, "tx_kib": [0] * 18,
            "rx_kib": [0] * 18, "errors": [[0, 0, 0] for _ in range(18)], "failed_fields": [0] * 18,
            "remote_bus_id": [""] * 18}


def test_counters_advance_by_the_scripted_step_on_their_own_device_and_link(tmp_path, sampler):
    """Each scripted field moves by its step between the two samples, on exactly its device, link and direction, and
    every other field stays 0: a sampler that dropped the scopeId would read one value for every link, and one that
    took the samples in the wrong order would read nothing."""
    rows = sampler(tmp_path, f"""\
        gpus 4
        field 1 7 {TX} 1000 4096
        field 1 7 {RX} 50 3
        field 1 8 {TX} 7 1
        field 2 0 {RX} 123456789 65536
        field 2 17 {TX} 9 0
        """, [fake_uuid(g) for g in (0, 1, 2)])
    want = [clean(), clean(), clean()]
    want[1]["tx_kib"][7], want[1]["rx_kib"][7], want[1]["tx_kib"][8] = 4096, 3, 1
    want[2]["rx_kib"][0] = 65536
    assert rows == want


def test_a_link_lost_between_samples(tmp_path, sampler):
    rows = sampler(tmp_path, "gpus 2\nlink_down 1 3\nlink_down_after 1 11\n", [fake_uuid(0), fake_uuid(1)])
    assert rows[0] == clean()
    want = clean(((1 << 18) - 1) & ~(1 << 3))
    want["lost_mask"] = 1 << 11
    assert rows[1] == want


def test_error_counters_rise_on_one_link_only(tmp_path, sampler):
    rows = sampler(tmp_path, f"""\
        gpus 2
        field 1 7 {REPLAY} 10 312
        field 1 7 {CRC} 0 41
        field 1 7 {RECOVERY} 5 0
        field 1 6 {REPLAY} 99 0
        """, [fake_uuid(0), fake_uuid(1)])
    want = clean()
    want["errors"][7] = [312, 0, 41]
    want["error_mask"] = 1 << 7
    assert rows == [clean(), want]
    assert links_ref.delta(*[{"status": 0, "link_mask": (1 << 18) - 1, "failed": [0] * 18, "remote": [""] * 18,
                              "value": [[0, 0, 10 + 312 * k, 5, 41 * k] if l == 7 else [0] * 5 for l in range(18)]}
                             for k in (0, 1)]) == want


def test_a_pcie_card_and_a_failing_field(tmp_path, sampler):
    """Every field NOT_SUPPORTED is a GPU without NVLink: status CDPROBE_ERR_UNSUPPORTED and nothing else.  One field
    that fails marks that field of that link only; the call failing as a whole is its nvmlReturn_t."""
    rows = sampler(tmp_path, "gpus 1\nunsupported nvlink\n", [fake_uuid(0)])
    assert rows == [dict(clean(0), status=links_ref.ERR_UNSUPPORTED)]
    rows = sampler(tmp_path, f"gpus 2\nfield_fail 1 4 {RECOVERY} {UNKNOWN}\nfield 1 4 {TX} 0 8\n",
                   [fake_uuid(0), fake_uuid(1)])
    want = clean()
    want["failed_fields"][4] = 0x08
    want["tx_kib"][4] = 8
    assert rows == [clean(), want]
    rows = sampler(tmp_path, f"gpus 1\nfail fields {UNKNOWN}\n", [fake_uuid(0)])
    assert rows == [dict(clean(0), status=UNKNOWN)]


def test_unknown_uuid_mig_and_missing_nvml(tmp_path, sampler):
    rows = sampler(tmp_path, "gpus 2\n", [fake_uuid(1), "GPU-not-there", "MIG:" + fake_uuid(0)])
    assert rows[0] == clean()
    assert rows[1] == dict(clean(0), status=6)  # NVML_ERROR_NOT_FOUND
    assert rows[2] == dict(clean(0), status=links_ref.ERR_UNSUPPORTED)
    rows = sampler(tmp_path, "gpus 1\n", [fake_uuid(0)], nvml="/nonexistent/libnvidia-ml.so.1")
    assert rows == [dict(clean(0), status=links_ref.ERR_UNSUPPORTED)]
    rows = sampler(tmp_path, "gpus 1\nfail init 9\n", [fake_uuid(0)])
    assert rows == [dict(clean(0), status=9)]


def test_remote_bus_ids(tmp_path, sampler):
    rows = sampler(tmp_path, "gpus 2\nremote 1 0 00000000:05:00.0\nremote 1 17 00000000:A3:00.0\nremote 0 2 x\n"
                   "link_down 0 2\n", [fake_uuid(0), fake_uuid(1)])
    assert rows[0]["remote_bus_id"] == [""] * 18  # link 2 is down: its remote is not asked for
    assert rows[1]["remote_bus_id"][0] == "00000000:05:00.0" and rows[1]["remote_bus_id"][17] == "00000000:A3:00.0"
    assert rows[1]["remote_bus_id"][1:17] == [""] * 16


# ---- the C++ daemon against the library test double --------------------------------------------------------------
@pytest.fixture(scope="module")
def fake_lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("fakelib")
    full, bare = d / "libfake_cdprobe.so", d / "libfake_cdprobe_nolinks.so"
    src = os.path.join(ROOT, "tests", "c")
    subprocess.run(["gcc", "-shared", "-fPIC", "-O1", "-Wall", os.path.join(src, "fake_cdprobe_links.c"), "-o",
                    str(full)], check=True)
    subprocess.run(["gcc", "-shared", "-fPIC", "-O1", "-Wall", os.path.join(src, "fake_cdprobe.c"), "-o", str(bare)],
                   check=True)
    return {"full": str(full), "bare": str(bare)}


def daemon_once(pkg, tmp_path, lib, links_script="", flag=None):
    env = dict(os.environ, CDPROBE_LIBRARY=lib, COMPUTE_DOMAIN_UUID="cd-1", FAKE_CDPROBE_SCRIPT="ok",
               FABRIC_PROBE_VERDICT_PATH=str(tmp_path / "v.json"), FABRIC_PROBE_METRICS_PATH=str(tmp_path / "m.prom"),
               FAKE_CDPROBE_LINKS=links_script, NODE_NAME="node-a", FAKE_CDPROBE_LOG=str(tmp_path / "calls.log"))
    env.pop("FABRIC_PROBE_LINK_COUNTERS", None)
    if flag is not None:
        env["FABRIC_PROBE_LINK_COUNTERS"] = flag
    exe = os.path.join(os.path.dirname(pkg.build.LIB), "cdprobe-daemon")
    r = subprocess.run([exe, "run", "--once"], env=env, capture_output=True, text=True, timeout=60)
    lines = [l for l in r.stderr.splitlines() if l.startswith("fabric probe links:")]
    prom = (tmp_path / "m.prom").read_text()
    log = tmp_path / "calls.log"
    calls = log.read_text().split("\n") if log.exists() else []
    return r, lines, prom, calls


def test_daemon_flag_off_logs_and_exports_nothing(pkg, tmp_path, fake_lib):
    r, lines, prom, calls = daemon_once(pkg, tmp_path, fake_lib["full"], "error")
    assert r.returncode == 0 and lines == []
    assert "fabric_probe_link" not in prom
    assert not any(c.startswith("set_option") for c in calls)


def test_daemon_flag_on_clean_pass_exports_series_without_a_line(pkg, tmp_path, fake_lib):
    r, lines, prom, calls = daemon_once(pkg, tmp_path, fake_lib["full"], "clean", "true")
    assert r.returncode == 0 and lines == []
    assert "set_option 27 1" in calls
    assert "# TYPE nvidia_dra_fabric_probe_link_kib gauge" in prom
    assert "# TYPE nvidia_dra_fabric_probe_link_errors gauge" in prom
    assert ('nvidia_dra_fabric_probe_link_kib{node="node-a",gpu="GPU-fa4e0000-0000-0000-0000-000000000000",link="0",'
            'dir="tx"} 1024') in prom
    assert ('nvidia_dra_fabric_probe_link_errors{node="node-a",gpu="GPU-fa4e0000-0000-0000-0000-000000000001",'
            'link="17",counter="crc"} 0') in prom
    series = [l for l in prom.splitlines() if l.startswith("nvidia_dra_fabric_probe_link_")]
    assert len(series) == 2 * 18 * 2 + 2 * 18 * 3  # two GPUs, every link: tx and rx, three error counters
    v = json.loads((tmp_path / "v.json").read_text())
    assert "links" not in json.dumps(sorted(v))  # the verdict file does not change


def test_daemon_logs_an_error_and_a_lost_link_exactly(pkg, tmp_path, fake_lib):
    r, lines, prom, _ = daemon_once(pkg, tmp_path, fake_lib["full"], "error", "1")
    assert r.returncode == 0
    assert lines == ["fabric probe links: GPU-fa4e0000-0000-0000-0000-000000000001 link 7 (remote 0000:05:00.0): "
                     "replay +312 recovery +0 crc +41; link 11 lost"]
    assert ('nvidia_dra_fabric_probe_link_errors{node="node-a",gpu="GPU-fa4e0000-0000-0000-0000-000000000001",'
            'link="7",counter="replay"} 312') in prom
    assert "fabric probe: verdict ok" in r.stderr


def test_daemon_without_cdprobe_links_runs_the_pass_unaffected(pkg, tmp_path, fake_lib):
    r, lines, prom, calls = daemon_once(pkg, tmp_path, fake_lib["bare"], "error", "true")
    assert r.returncode == 0 and lines == []
    assert "fabric_probe_link" not in prom
    assert "fabric probe: verdict ok" in r.stderr
    assert json.loads((tmp_path / "v.json").read_text())["ok"] is True
