"""The bench.py JSON contract: every key a consumer reads is present with the right type and the numbers are
internally consistent.  Checked on a live line on the GPU; the parity self-check's logic is checked on CPU."""
import json
import os

import pytest

from conftest import ROOT

REQUIRED = {"metric": str, "value": float, "unit": str, "n_gpus": int, "steps": int, "warmup": int,
            "ms_per_step": float, "higher_is_better": bool, "scaling": str, "dtype": str, "data": str, "config": dict,
            "e2e": dict, "gpu_launches": int, "roofline": dict, "clocks": dict}


# ---- the parity self-check of bench.py is not vacuous: a wrong checksum or a wrong reach bit is caught -------------
def test_parity_block_catches_mismatches(pkg, oracle, monkeypatch):
    import types

    import bench

    n, nbytes, mode = 3, 3 << 12, 1
    bpp = oracle.plan(n, nbytes, mode).bytes_per_pair
    words = bpp // 8
    seed, run_seq = oracle.DEFAULT_SEED, 7

    def result():
        r = types.SimpleNamespace(bytes_per_pair=bpp, run_seq=run_seq)
        z = [[0] * n for _ in range(n)]
        r.sum_read, r.xor_read, r.sum_write, r.xor_write = ([row[:] for row in z] for _ in range(4))
        r.reach = [[1] * n for _ in range(n)]
        for i in range(n):
            for j in range(n):
                if i != j:
                    r.sum_read[i][j], r.xor_read[i][j] = oracle.expected_read(seed, n, nbytes, mode, i, j)
                    r.sum_write[i][j], r.xor_write[i][j] = oracle.write_checksum(seed, i, j, run_seq, words)
        return r

    # no NVML in this container: the reach half must say so (None), never assume
    good = bench.parity_block(pkg, oracle, result(), n, nbytes, mode, [f"GPU-{i}" for i in range(n)], seed)
    assert good["cells"] == 6 and good["checksum_ok"] is True and good["reach_vs_nvml_ok"] is None and good["reach_vs_nvml_error"]
    bad = result()
    bad.xor_write[2][0] ^= 1 << 40
    blk = bench.parity_block(pkg, oracle, bad, n, nbytes, mode, [f"GPU-{i}" for i in range(n)], seed)
    assert blk["checksum_ok"] is False and blk["checksum_mismatches"] == [["write", 2, 0]]
    # with an NVML that answers (the fake one): an unreachable cell the NVML poll calls reachable is a parity failure
    fake = types.SimpleNamespace(uuids=lambda: [f"GPU-{i}" for i in range(n)], reach_matrix=lambda: [[1] * n for _ in range(n)], n=n)
    monkeypatch.setattr(oracle, "nvml_poll", lambda *a, **k: fake)
    r = result()
    assert bench.parity_block(pkg, oracle, r, n, nbytes, mode, [f"GPU-{i}" for i in (2, 0, 1)], seed)["reach_vs_nvml_ok"] is True
    r.reach[1][2] = 0
    blk = bench.parity_block(pkg, oracle, r, n, nbytes, mode, [f"GPU-{i}" for i in range(n)], seed)
    assert blk["reach_vs_nvml_ok"] is False and blk["reach_mismatches"] == [[1, 2, 0, 1]]


@pytest.mark.gpu
def test_bench_runs_end_to_end_with_parity(tmp_path, oracle):
    """bench.py itself on the GPU (N = 1, a few steps): exit 0, one JSON line with the full schema, parity block
    green, roofline against the peak, and --dump-outputs holding exactly what the last timed step returned."""
    import subprocess
    import sys

    import numpy as np

    dump = tmp_path / "dump"
    cp = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "10", "--warmup", "3",
                         "--no-cpu-baseline", "--no-daemon", "--dump-outputs", str(dump)],
                        capture_output=True, text=True, timeout=300)
    assert cp.returncode == 0, cp.stderr[-2000:]
    lines = [l for l in cp.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    j = json.loads(lines[0])
    for k, t in REQUIRED.items():
        assert k in j, k
        assert isinstance(j[k], t) or (t is float and isinstance(j[k], int)), (k, type(j[k]))
    assert j["metric"] == "nvlink_probe_ms" and j["unit"] == "ms" and j["higher_is_better"] is False
    assert j["vs_baseline"] is None and j["data"] == "synthetic" and j["scaling"] == "weak" and j["warmup"] >= 3
    assert j["n_gpus"] == 1 and j["steps"] == 10 and j["gpu_launches"] == 10 and j["parity"]["checksum_ok"] is True
    assert j["parity"]["reach_vs_nvml_ok"] is True and j["verdict"] is True and 0.5 < j["roofline"]["frac"] < 1.1
    assert "workload" in j["config"] and "model" not in j["config"]
    assert j["value"] >= j["kernel_ms_globaltimer"] >= j["device_ms_globaltimer"] > 0
    e = j["e2e"]
    assert e["unit"] == "ms" and e["value"] > 0 and e["d2h_bytes_per_step"] == 48 + 120 * j["config"]["phases"]
    r = j["roofline"]
    assert r["bound"] == "hbm" and set(["bound", "achieved", "peak", "unit", "frac", "traffic"]) <= set(r)
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9 and r["unit"] == "GB/s"
    assert not set(j["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    assert j["reachability_all_ones"] is True
    # the dump: float arrays only, the cell's reach bits and its 64-bit checksums as exact (high, low) halves
    names = sorted(p.name for p in dump.iterdir())
    assert names == sorted(f"{n}.npy" for n in ("reach_read", "reach_write", "status", "sum_read", "xor_read",
                                                "sum_write", "xor_write"))
    arrs = {p.stem: np.load(p) for p in dump.iterdir()}
    assert all(a.dtype in (np.float32, np.float64) for a in arrs.values())
    assert arrs["reach_read"].tolist() == [[1.0]] and arrs["reach_write"].tolist() == [[1.0]]
    assert arrs["status"].tolist() == [[0.0]]

    def u64(name):
        hi, lo = arrs[name][0, 0]
        return (int(hi) << 32) | int(lo)

    nbytes, words = 1 << 30, (1 << 30) // 8
    assert (u64("sum_read"), u64("xor_read")) == oracle.expected_read(oracle.DEFAULT_SEED, 1, nbytes, 1, 0, 0)
    # the write pattern is salted with the run counter: the open-time pass, 1 + warm-up + 1 + steps + 1 + steps runs
    run_seq = 1 + 1 + j["warmup"] + 1 + 10 + 1 + 10
    assert (u64("sum_write"), u64("xor_write")) == oracle.write_checksum(oracle.DEFAULT_SEED, 0, 0, run_seq, words)
