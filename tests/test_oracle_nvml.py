"""Known-answer tests of the NVML oracle (oracle/nvml_poll.c) against the scriptable fake
libnvidia-ml.so.1 (tests/fake_nvml).  Scenario list: SURVEY.md §8(c) / Appendix C tier T1.

Each oracle call runs in a fresh process so the fake library re-reads its scenario.
"""
import json
import os
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = os.path.join(ROOT, "tests", "fake_nvml", "libnvidia-ml.so.1")

CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    from oracle import oracle as o
    rc, r = o.nvml_poll_rc(int(sys.argv[1]), int(sys.argv[2]))
    n = r.n
    print(json.dumps({
        "rc": rc, "n": n, "reach": r.reach_matrix(), "n_links": list(r.n_links)[:n],
        "link_mask": [sum(1 << l for l in range(18) if r.link_active[i][l]) for i in range(n)],
        "mig": list(r.mig_enabled)[:n], "clique_id": r.clique_id.decode(), "clique_err": r.clique_err,
        "clique_err_text": r.clique_err_text.decode(), "imex_gate": r.imex_gate, "calls": r.nvml_calls,
        "uuids": r.uuids(), "name0": r.name[0].value.decode() if n else "", "cc": [r.cc_major[0], r.cc_minor[0]],
        "total_ms": r.total_ms,
    }))
    """
) % ROOT


def poll(tmp_path, scenario: str, n_max=0, flags=0, env_extra=None, nvml_path=FAKE):
    sc = tmp_path / "scenario.txt"
    sc.write_text(scenario)
    env = dict(os.environ)
    env["FAKE_NVML_SCENARIO"] = str(sc)
    env["CDORACLE_NVML_PATH"] = nvml_path
    env.pop("CLIQUE_ID", None)
    env.update(env_extra or {})
    out = subprocess.run([sys.executable, "-c", CHILD, str(n_max), str(flags)], env=env, capture_output=True,
                         text=True, timeout=60)
    assert out.returncode == 0, out.stderr
    return json.loads(out.stdout.strip().splitlines()[-1])


def identity(n):
    return [[1 if i == j else 0 for j in range(n)] for i in range(n)]


def ones(n):
    return [[1] * n for _ in range(n)]


@pytest.fixture(scope="module", autouse=True)
def _built(oracle):
    assert os.path.exists(FAKE)


def test_all_up_8_gpus(tmp_path):
    r = poll(tmp_path, "gpus 8\n")
    assert r["rc"] == 0 and r["n"] == 8
    assert r["reach"] == ones(8)
    assert r["n_links"] == [18] * 8
    # single-node HGX: zero cluster UUID => no clique, the IMEX gate does not apply (SURVEY F7)
    assert r["clique_id"] == "" and r["clique_err"] == 0 and r["imex_gate"] == -1
    # call budget of SURVEY §8(d): 144 link polls + 168 P2P polls + enumerate/fabric/lifecycle
    assert r["calls"] >= 144 + 168
    assert r["cc"] == [9, 0]


def test_one_link_down_keeps_gpu_reachable(tmp_path):
    r = poll(tmp_path, "gpus 8\nlink_down 3 5\n")
    assert r["n_links"][3] == 17
    assert r["reach"] == ones(8)


def test_all_links_down_on_one_gpu(tmp_path):
    sc = "gpus 4\n" + "".join(f"link_down 2 {l}\n" for l in range(18))
    r = poll(tmp_path, sc)
    exp = ones(4)
    for k in range(4):
        if k != 2:
            exp[2][k] = exp[k][2] = 0
    assert r["reach"] == exp


def test_p2p_disabled_for_one_ordered_pair(tmp_path):
    # NVML_P2P_STATUS_DISABLED_BY_REGKEY == 6 for (2,5) only: the matrix is not symmetric
    r = poll(tmp_path, "gpus 8\np2p 2 5 nvlink 6\n")
    exp = ones(8)
    exp[2][5] = 0
    assert r["reach"] == exp
    r = poll(tmp_path, "gpus 8\np2p 2 5 read 3\np2p 5 2 write 4\n")
    exp = ones(8)
    exp[2][5] = exp[5][2] = 0
    assert r["reach"] == exp


def test_mig_enabled_gpu_has_no_peers(tmp_path):
    r = poll(tmp_path, "gpus 8\nmig 6 1\n")
    exp = ones(8)
    for k in range(8):
        if k != 6:
            exp[6][k] = exp[k][6] = 0
    assert r["reach"] == exp and r["mig"][6] == 1


def test_all_mig_is_identity(tmp_path):
    # config 4: 8 MIG instances => identity matrix (SURVEY F7 / H8)
    r = poll(tmp_path, "gpus 8\n" + "".join(f"mig {g} 1\n" for g in range(8)))
    assert r["reach"] == identity(8)


def test_everything_not_supported(tmp_path):
    r = poll(tmp_path, "gpus 4\nunsupported nvlink\nunsupported p2p\nunsupported fabric\nunsupported mig\n")
    assert r["rc"] == 0
    assert r["reach"] == identity(4)  # NOT_SUPPORTED => predicate false, not an error
    assert r["clique_id"] == "" and r["clique_err"] == 0


def test_single_gpu(tmp_path):
    r = poll(tmp_path, "gpus 1\n")
    assert r["n"] == 1 and r["reach"] == [[1]]


def test_n_max_clamps(tmp_path):
    r = poll(tmp_path, "gpus 8\n", n_max=2)
    assert r["n"] == 2 and r["reach"] == ones(2)


def test_sixteen_gpus(tmp_path):
    r = poll(tmp_path, "gpus 16\n")
    assert r["n"] == 16 and r["reach"] == ones(16)


def test_uuid_order_differs_from_index_order(tmp_path):
    a = poll(tmp_path, "gpus 4\n")
    b = poll(tmp_path, "gpus 4\nuuid_reverse\n")
    assert a["uuids"] == list(reversed(b["uuids"]))


UUID = "00112233445566778899aabbccddeeff"
UUID_S = "00112233-4455-6677-8899-aabbccddeeff"


def test_clique_id_strict_mnnvl(tmp_path):
    # getCliqueIDStrict: state COMPLETED(3), status 0, non-zero cluster UUID, all GPUs agree
    r = poll(tmp_path, f"gpus 4\nfabric_all 3 0 7 {UUID}\n")
    assert r["clique_id"] == f"{UUID_S}.7" and r["clique_err"] == 0


def test_clique_id_strict_in_progress_is_an_error(tmp_path):
    # nvlib.go:309-311: fabric supported but registration not completed => refuse to start
    r = poll(tmp_path, f"gpus 4\nfabric_all 3 0 7 {UUID}\nfabric 2 2 0 7 {UUID}\n")
    assert r["clique_err"] != 0 and "state=2" in r["clique_err_text"] and r["clique_id"] == ""


def test_clique_id_legacy_in_progress_is_skipped(tmp_path):
    # IsFabricAttached: not COMPLETED => "not attached", device skipped, others still form the clique
    r = poll(tmp_path, f"gpus 4\nfabric_all 3 0 7 {UUID}\nfabric 2 2 0 7 {UUID}\n", flags=1)
    assert r["clique_err"] == 0 and r["clique_id"] == f"{UUID_S}.7"


def test_clique_id_strict_status_error(tmp_path):
    r = poll(tmp_path, f"gpus 2\nfabric_all 3 0 7 {UUID}\nfabric 1 3 999 7 {UUID}\n")
    assert r["clique_err"] != 0 and "registration error" in r["clique_err_text"]


def test_clique_id_mismatch_is_an_error(tmp_path):
    r = poll(tmp_path, f"gpus 2\nfabric_all 3 0 7 {UUID}\nfabric 1 3 0 8 {UUID}\n")
    assert r["clique_err"] != 0 and "CliqueIDs" in r["clique_err_text"]
    other = "ff" + UUID[2:]
    r = poll(tmp_path, f"gpus 2\nfabric_all 3 0 7 {UUID}\nfabric 1 3 0 7 {other}\n")
    assert r["clique_err"] != 0 and "ClusterUUIDs" in r["clique_err_text"]


def test_fabric_state_not_supported_means_no_clique(tmp_path):
    r = poll(tmp_path, f"gpus 2\nfabric_all 0 0 0 {'00' * 16}\n")
    assert r["clique_id"] == "" and r["clique_err"] == 0


def _fake_imex_ctl(tmp_path, text, code=0):
    p = tmp_path / "nvidia-imex-ctl"
    p.write_text(f"#!/bin/sh\nprintf '{text}'\nexit {code}\n")
    p.chmod(0o755)
    return str(p)


def test_imex_gate_ready(tmp_path):
    ctl = _fake_imex_ctl(tmp_path, "READY\\n")
    r = poll(tmp_path, "gpus 4\n", env_extra={"CLIQUE_ID": f"{UUID_S}.7", "CDORACLE_IMEX_CTL": ctl})
    assert r["imex_gate"] == 1 and r["reach"] == ones(4)


@pytest.mark.parametrize("text,code", [("NOT_READY\\n", 0), ("READY", 0), ("READY\\n", 1), ("READY\\nextra\\n", 0)])
def test_imex_gate_not_ready_clears_off_diagonal(tmp_path, text, code):
    # main.go:448-456: anything but exit 0 + exactly "READY\n" fails the check
    ctl = _fake_imex_ctl(tmp_path, text, code)
    r = poll(tmp_path, "gpus 4\n", env_extra={"CLIQUE_ID": f"{UUID_S}.7", "CDORACLE_IMEX_CTL": ctl})
    assert r["imex_gate"] == 0 and r["reach"] == identity(4)


def test_imex_gate_noop_without_clique(tmp_path):
    # main.go:436-439: CLIQUE_ID == "" => check is a no-op
    ctl = _fake_imex_ctl(tmp_path, "NOT_READY\\n")
    r = poll(tmp_path, "gpus 4\n", env_extra={"CLIQUE_ID": "", "CDORACLE_IMEX_CTL": ctl})
    assert r["imex_gate"] == -1 and r["reach"] == ones(4)


@pytest.mark.parametrize("scenario", ["gpus 8\n", "gpus 8\nlink_down 3 5\nmig 6 1\np2p 2 5 nvlink 6\n", "gpus 1\n",
                                      "gpus 16\np2p 0 15 read 3\n"])
def test_threaded_poll_gives_the_same_answer(tmp_path, scenario):
    """The N-thread variant of the link/P2P polls (one worker per GPU) is only a timing variant."""
    a = poll(tmp_path, scenario, flags=0)
    b = poll(tmp_path, scenario, flags=8)
    for k in ("rc", "n", "reach", "n_links", "mig", "clique_id", "calls", "uuids"):
        assert a[k] == b[k], k


def test_nvml_missing_is_a_clean_error(tmp_path):
    r = poll(tmp_path, "gpus 4\n", nvml_path="/nonexistent/libnvidia-ml.so.1")
    assert r["rc"] == -1


def test_init_failure_is_reported(tmp_path):
    r = poll(tmp_path, "gpus 4\nfail init 9\n")  # NVML_ERROR_DRIVER_NOT_LOADED
    assert r["rc"] == 9


# ---- the product's topology enumeration (csrc/topo.cc) must agree with the oracle ----------
TOPO_CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    try:
        t = m.topology(strict=bool(int(sys.argv[1])))
        print(json.dumps({"rc": 0, "n": t.n, "uuids": [t.uuid[i].value.decode() for i in range(t.n)],
                          "mig": list(t.mig)[:t.n], "links": list(t.links_active)[:t.n],
                          "link_mask": list(t.link_mask)[:t.n],
                          "clique_id": t.clique_id.decode(), "clique_error": t.clique_error.decode(),
                          "pci": [t.pci_bus_id[i].value.decode() for i in range(t.n)]}))
    except m.ProbeError as e:
        print(json.dumps({"rc": e.code}))
    """
) % ROOT


def topo(tmp_path, scenario, strict=1, nvml_path=FAKE):
    sc = tmp_path / "scenario.txt"
    sc.write_text(scenario)
    env = dict(os.environ, FAKE_NVML_SCENARIO=str(sc), CDPROBE_NVML_PATH=nvml_path)
    out = subprocess.run([sys.executable, "-c", TOPO_CHILD, str(strict)], env=env, capture_output=True, text=True,
                         timeout=60)
    assert out.returncode == 0, out.stderr
    return json.loads(out.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("scenario", [
    "gpus 8\n", "gpus 8\nlink_down 3 5\nmig 6 1\n", "gpus 4\nuuid_reverse\n", "gpus 1\n", "gpus 16\n",
    f"gpus 4\nfabric_all 3 0 7 {UUID}\n", f"gpus 4\nfabric_all 3 0 7 {UUID}\nfabric 2 2 0 7 {UUID}\n",
    f"gpus 2\nfabric_all 3 0 7 {UUID}\nfabric 1 3 0 8 {UUID}\n", "gpus 4\nunsupported fabric\nunsupported nvlink\n",
    f"gpus 2\nfabric_all 3 0 7 {UUID}\nfabric 1 3 999 7 {UUID}\n",
])
@pytest.mark.parametrize("strict", [1, 0])
def test_product_topology_agrees_with_oracle(pkg, tmp_path, scenario, strict):
    """Parity of the host-side mirror of getCliqueID*/device walk: same UUID order, MIG flags, link counts,
    clique id and error class as the oracle restatement, on every fake-NVML scenario."""
    t = topo(tmp_path, scenario, strict)
    o = poll(tmp_path, scenario, flags=0 if strict else 1)
    assert t["rc"] == 0 and o["rc"] == 0
    assert t["n"] == o["n"] and t["uuids"] == o["uuids"]
    assert t["mig"] == o["mig"] and t["links"] == o["n_links"]
    assert t["link_mask"] == o["link_mask"]  # WHICH physical link is down, not only how many are up
    assert all(bin(m).count("1") == k for m, k in zip(t["link_mask"], t["links"]))
    assert t["clique_id"] == o["clique_id"]
    assert bool(t["clique_error"]) == bool(o["clique_err"])
    if t["clique_error"]:
        assert t["clique_error"] == o["clique_err_text"]


def test_product_topology_without_nvml_fails_loudly(pkg, tmp_path):
    t = topo(tmp_path, "gpus 2\n", nvml_path="/nonexistent/libnvidia-ml.so.1")
    assert t["rc"] == -3  # CDPROBE_ERR_NO_DEVICE
