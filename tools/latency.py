#!/usr/bin/env python3
"""Dependent-load latency of cdprobe_latency on one GPU, ns per hop (min / median / max over the timed reps):
  - N = 1 loop-back at regions of 64 KiB (L2-resident), 64 MiB and 1 GiB;
  - two ranks on the same device (N = 2): cells (0, 1) and (1, 0) through a second VMM mapping of the same HBM.
Every chase's digest is checked by the library (status 0).  This is local L2 / HBM latency through a VMM mapping;
latency over NVLink needs two GPUs and is not measured here.
Prints one JSON document with the card's name, power limit and SM clock read in the same call (read-only query)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cdprobe_pkg  # noqa: E402

pkg = cdprobe_pkg.load()
ap = argparse.ArgumentParser()
ap.add_argument("--hops", type=int, default=4096)
ap.add_argument("--reps", type=int, default=32)
ap.add_argument("--out", default=None, help="also write the JSON document to this file")
a = ap.parse_args()


def gpu():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def cell(lat, i, j):
    assert lat.measured[i][j] and lat.status[i][j] == 0, (i, j, lat.status[i][j])
    return {"ns_min": lat.ns_min[i][j], "ns_median": lat.ns_median[i][j], "ns_max": lat.ns_max[i][j]}


res = {"hops": a.hops, "reps": a.reps, "what": "ns per dependent 8-byte ld.relaxed.sys load through a VMM mapping of "
       "local HBM, one untimed warm-up rep first"}
for name, nbytes in (("n1_64KiB", 64 << 10), ("n1_64MiB", 64 << 20), ("n1_1GiB", 1 << 30)):
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes)) as p:
        lat = p.Latency(a.hops, a.reps)
        res[name] = {"region_bytes": lat.region_bytes, **cell(lat, 0, 0), "call_ms": lat.ms}
SAME = pkg.abi.FLAG_ALLOW_SAME_DEVICE | pkg.abi.FLAG_NO_COOPERATIVE
with pkg.Open(pkg.Config(ordinals=[0, 0], bytes=1 << 30, flags=SAME, ctas=16, timeout_ms=20000)) as p:
    lat = p.Latency(a.hops, a.reps)
    res["n2_same_device"] = {"region_bytes": lat.region_bytes, "cell_0_1": cell(lat, 0, 1), "cell_1_0": cell(lat, 1, 0),
                             "call_ms": lat.ms}
res["gpu"] = gpu()
res["nvlink"] = "not measured (one GPU)"
if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
print(json.dumps(res, indent=1))
