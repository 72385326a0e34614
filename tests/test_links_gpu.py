"""cdprobe_links on the device (DESIGN §5o): the option is off by default and then loads no NVML, the same pass reads
the same with and without it, the samples stay outside probe_ms, and the rows, masks and expected payload are right for
one GPU, for ranks that share a GPU in one process and in two, and across GPUs where there are several.

The machines are shared: another tenant's traffic can move a GPU's NVLink counters, so no test asserts zero observed
traffic.  The observed deltas are printed ("LINKS ..." lines) and asserted only where payload must have crossed."""
import json
import os
import subprocess
import sys
import textwrap
import uuid

import pytest

from conftest import ROOT, gpu_count
from test_links_cpu import build_fake_nvml

pytestmark = pytest.mark.gpu

NGPU = gpu_count()
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
NBYTES = 64 << 20
SEED = 0x5EED11


def record(what, **kw):
    print("LINKS " + json.dumps(dict(test=what, **kw)))


def run_child(code, *args, env=None, timeout=300):
    out = subprocess.run([sys.executable, "-c", code, *map(str, args)], capture_output=True, text=True, timeout=timeout,
                         env=env)
    assert out.returncode == 0, out.stderr[-3000:]
    return json.loads([l for l in out.stdout.splitlines() if l.startswith("RESULT ")][-1][7:])


HEAD = "import json, sys\nsys.path.insert(0, %r)\nimport cdprobe_pkg\npkg = cdprobe_pkg.load()\n" % ROOT


OFF_CHILD = HEAD + textwrap.dedent("""
    def nvml_maps():
        return sorted({l.split()[-1] for l in open("/proc/self/maps") if "libnvidia-ml" in l})
    before = nvml_maps()
    assert "torch" not in sys.modules and "pynvml" not in sys.modules
    with pkg.Open(pkg.Config(ordinals=[0], bytes=%d)) as p:
        r = p.Run()
        links = p.Links()
        during = nvml_maps()
    after = nvml_maps()
    assert "torch" not in sys.modules and "pynvml" not in sys.modules
    print("RESULT " + json.dumps({"before": before, "during": during, "after": after, "run_seq": r.run_seq,
                                  "links_seq": links.run_seq, "n_devices": links.n_devices,
                                  "zero": bytes(links.raw)[4:] == bytes(len(bytes(links.raw)) - 4)}))
""") % NBYTES


def test_off_by_default_loads_no_nvml_and_reports_nothing():
    """A process that never imports torch or pynvml opens, runs and closes a handle with the option left off: no
    libnvidia-ml mapping appears beyond those present before cdprobe_open, and cdprobe_links says no run was sampled."""
    r = run_child(OFF_CHILD)
    record("off_by_default", **r)
    assert set(r["during"]) <= set(r["before"]) and set(r["after"]) <= set(r["before"])
    assert r["run_seq"] >= 2 and r["links_seq"] == 0 and r["n_devices"] == 0 and r["zero"]


def open_one(pkg, on, **kw):
    p = pkg.Open(pkg.Config(ordinals=kw.pop("ordinals", [0]), bytes=kw.pop("nbytes", NBYTES), seed=SEED, **kw))
    if on:
        p.SetOption(pkg.abi.OPT_LINK_COUNTERS, 1)
    return p


def same_pass(a, b):
    n = a.n
    for f in ("reach_read", "reach_write", "status", "sum_read", "xor_read", "sum_write", "xor_write"):
        assert getattr(a, f) == getattr(b, f), f
    assert (a.verdict, a.run_seq, a.aborted, a.phases, n) == (b.verdict, b.run_seq, b.aborted, b.phases, b.n)


def link_mask_of(pkg, uuid_):
    t = pkg.fabricprobe.topology(strict=False)
    for i in range(t.n):
        if t.uuid[i].value.decode() == uuid_:
            return t.link_mask[i]
    return None


def test_the_same_pass_with_and_without_the_counters(pkg):
    """Same seed, a fresh handle each: reach bits, checksums, statuses and verdict are identical."""
    with open_one(pkg, False) as p:
        off = p.Run()
        assert p.Links().run_seq == 0
    with open_one(pkg, True) as p:
        on = p.Run()
        links = p.Links()
    same_pass(off, on)
    assert links.run_seq == on.run_seq


def test_one_gpu(pkg):
    with open_one(pkg, True) as p:
        info = p.Info()
        res = [p.Run() for _ in range(3)]
        links = p.Links()
    me = info.uuid[0].value.decode()
    assert links.run_seq == res[-1].run_seq and links.n_devices == 1
    d = links.devices[0]
    assert d["uuid"] == me and d["rank_mask"] == 1
    assert d["expected_tx_kib"] == 0 and d["expected_rx_kib"] == 0  # the loop-back never leaves the GPU
    assert links.sample_ms > 0
    if d["status"] == pkg.abi.ERR_UNSUPPORTED:
        case = "no NVLink fields on this GPU: CDPROBE_ERR_UNSUPPORTED, the run unaffected"
        assert d["link_mask"] == 0 and all(r.verdict for r in res)
    else:
        case = "NVLink fields present"
        assert d["status"] == 0, d["status"]
        assert d["link_mask"] == link_mask_of(pkg, me)
    print(f"case: {case}")
    record("one_gpu", case=case, status=d["status"], link_mask=d["link_mask"], lost_mask=d["lost_mask"],
           error_mask=d["error_mask"], tx_kib=d["tx_kib"], rx_kib=d["rx_kib"], errors=d["errors"],
           remote_bus_id=d["remote_bus_id"], sample_ms=links.sample_ms, probe_ms=res[-1].probe_ms)


def test_sample_ms_and_probe_ms_with_and_without(pkg):
    """The option's cost on one GPU, measured: probe_ms of the same configuration off and on (alternated, 1 GiB, 20
    runs each), and sample_ms.  Recorded, not gated: the samples are outside probe_ms by construction."""
    import statistics
    cfg = dict(nbytes=1 << 30)
    with open_one(pkg, False, **cfg) as off, open_one(pkg, True, **cfg) as on:
        off.Run(), on.Run()
        t_off, t_on, s = [], [], []
        for _ in range(20):
            t_off.append(off.Run().probe_ms)
            t_on.append(on.Run().probe_ms)
            s.append(on.Links().sample_ms)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    record("cost", gpu=q.stdout.strip(), probe_ms_off=statistics.median(t_off), probe_ms_on=statistics.median(t_on),
           sample_ms=statistics.median(s), probe_ms_off_all=t_off, probe_ms_on_all=t_on, sample_ms_all=s)


PLACEMENT_CHILD = HEAD + textwrap.dedent("""
    with pkg.Open(pkg.Config(ordinals=[0], bytes=%d)) as p:
        p.Run()
        p.SetOption(pkg.abi.OPT_LINK_COUNTERS, 1)
        r = p.Run()
        links = p.Links()
    print("RESULT " + json.dumps({"probe_ms": r.probe_ms, "sample_ms": links.sample_ms, "run_seq": r.run_seq,
                                  "links_seq": links.run_seq, "status": links.devices[0]["status"],
                                  "tx": links.devices[0]["tx_kib"][3]}))
""") % NBYTES


def test_the_samples_stay_outside_probe_ms(pkg, tmp_path):
    """Against the fake NVML, whose field call takes 200 ms: both samples take it, and probe_ms does not."""
    with pkg.Open(pkg.Config(ordinals=[0], bytes=NBYTES)) as p:
        me = p.Info().uuid[0].value.decode()
    sc = tmp_path / "scenario.txt"
    sc.write_text(f"gpus 1\nuuid_alias 0 {me}\nfield_delay_us 200000\nfield 0 3 138 100 7\n")
    env = dict(os.environ, CDPROBE_NVML_PATH=build_fake_nvml(tmp_path), FAKE_NVML_SCENARIO=str(sc))
    r = run_child(PLACEMENT_CHILD, env=env)
    record("placement", **r)
    assert r["status"] == 0 and r["tx"] == 7 and r["links_seq"] == r["run_seq"]
    assert r["sample_ms"] >= 400.0
    assert r["probe_ms"] < 100.0


@pytest.mark.parametrize("n", [2, 4, 8])
def test_ranks_sharing_one_gpu_share_one_row(pkg, n):
    with open_one(pkg, True, ordinals=[0] * n, flags=SAME, ctas=8) as p:
        r = p.Run()
        links = p.Links()
    assert links.run_seq == r.run_seq and links.n_devices == 1
    d = links.devices[0]
    assert d["rank_mask"] == (1 << n) - 1
    assert d["expected_tx_kib"] == 0 and d["expected_rx_kib"] == 0
    record(f"same_device_{n}", status=d["status"], tx_kib=sum(d["tx_kib"]), rx_kib=sum(d["rx_kib"]))


TWO_PROC_CHILD = HEAD + textwrap.dedent("""
    session, rank = sys.argv[1], int(sys.argv[2])
    cfg = pkg.Config(ordinals=[0], bytes=%d, world_size=2, rank=rank, session=session, flags=0x40, ctas=8,
                     timeout_ms=30000)
    with pkg.Open(cfg) as p:
        p.SetOption(pkg.abi.OPT_LINK_COUNTERS, 1)
        r = p.Run()
        links = p.Links()
    print("RESULT " + json.dumps({"run_seq": r.run_seq, "links": [links.run_seq, links.n_devices],
                                  "dev": {k: links.devices[0][k] for k in ("rank_mask", "expected_tx_kib",
                                                                           "expected_rx_kib", "status")}}))
""") % NBYTES


def test_two_processes_sharing_one_gpu_report_their_own_ranks():
    session = f"lk-{uuid.uuid4().hex[:12]}"
    procs = [subprocess.Popen([sys.executable, "-c", TWO_PROC_CHILD, session, str(r)], stdout=subprocess.PIPE,
                              stderr=subprocess.PIPE, text=True) for r in range(2)]
    outs = []
    for pr in procs:
        so, se = pr.communicate(timeout=300)
        assert pr.returncode == 0, se[-3000:]
        outs.append(json.loads([l for l in so.splitlines() if l.startswith("RESULT ")][-1][7:]))
    for rank, o in enumerate(outs):
        assert o["links"] == [o["run_seq"], 1]
        assert o["dev"]["rank_mask"] == 1 << rank
        assert o["dev"]["expected_tx_kib"] == 0 and o["dev"]["expected_rx_kib"] == 0


@pytest.mark.skipif(NGPU < 2, reason="needs two GPUs")
def test_across_gpus_payload_shows_on_some_link(pkg):
    """Every GPU whose expected payload is above 0 shows DATA deltas above 0 on some link.  The observed / expected
    ratio per GPU is recorded, not asserted: whether NVML's DATA counters equal the payload has not been measured."""
    n = min(NGPU, 8)
    with open_one(pkg, True, ordinals=list(range(n)), nbytes=1 << 30) as p:
        r = p.Run()
        links = p.Links()
    assert links.run_seq == r.run_seq and links.n_devices == n
    for d in links.devices:
        if d["status"] != 0:
            continue
        assert d["expected_tx_kib"] > 0 and d["expected_rx_kib"] > 0
        assert sum(d["tx_kib"]) > 0 and sum(d["rx_kib"]) > 0, d["uuid"]
        record("across_gpus", uuid=d["uuid"], tx_ratio=sum(d["tx_kib"]) / d["expected_tx_kib"],
               rx_ratio=sum(d["rx_kib"]) / d["expected_rx_kib"], errors=d["errors"], lost=d["lost_mask"])
