#!/usr/bin/env python3
"""Cost of cdprobe_diagnose on one GPU: CUDA-event time (clear + compare pass + sample pass) of
  - a clean 1 GiB local region (read and write cell of the N = 1 loop-back after a passing run);
  - a 1 GiB write cell that is 100 % STALE (two ranks on one device; the pair is unmapped after a passing run, so the
    slot keeps the previous run's pattern and every word takes the classification path).
Prints one JSON document with the card's name, power limit and SM clock read in the same call."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cdprobe_pkg  # noqa: E402

pkg = cdprobe_pkg.load()
ap = argparse.ArgumentParser()
ap.add_argument("--bytes", type=int, default=1 << 30)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--out", default=None, help="also write the JSON document to this file")
a = ap.parse_args()


def timed(p, op, i, j, reader, expect_bad):
    for _ in range(3):
        p.Diagnose(op, i, j, reader)
    ms = []
    for _ in range(a.reps):
        d = p.Diagnose(op, i, j, reader)
        assert d.bad_words == expect_bad(d), (op, d.bad_words)
        ms.append(d.ms)
    return {"bytes": d.bytes, "bad_words": d.bad_words, "kinds": d.kinds, "reps": a.reps,
            "median_ms": statistics.median(ms), "min_ms": min(ms), "max_ms": max(ms),
            "median_gbps": d.bytes / statistics.median(ms) / 1e6}


def gpu():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_event_reasons.active"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


res = {}
with pkg.Open(pkg.Config(ordinals=[0], bytes=a.bytes)) as p:
    assert p.Run().verdict
    res["clean_read_local"] = timed(p, "read", 0, 0, 0, lambda d: 0)
    res["clean_write_local"] = timed(p, "write", 0, 0, 0, lambda d: 0)
    res["gpu_after_clean"] = gpu()
SAME = pkg.abi.FLAG_ALLOW_SAME_DEVICE | pkg.abi.FLAG_NO_COOPERATIVE
with pkg.Open(pkg.Config(ordinals=[0, 0], bytes=a.bytes, flags=SAME, ctas=16, timeout_ms=20000)) as p:
    assert p.Run().verdict
    p.UnmapPeer(0, 1)
    p.Run()
    res["stale_write_local"] = timed(p, "write", 0, 1, 1, lambda d: d.bytes // 8)
    assert res["stale_write_local"]["kinds"]["stale"] == res["stale_write_local"]["bytes"] // 8
    res["gpu_after_stale"] = gpu()
res["nvlink"] = "not measured (one GPU)"
if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
print(json.dumps(res, indent=1))
