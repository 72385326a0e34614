#!/usr/bin/env python3
"""Signal round trip of cdprobe_pingpong on one GPU, ns per round trip (min / median / max over the timed reps):
  - two ranks on the same device (N = 2): cells (0, 1) and (1, 0);
  - four ranks on the same device (N = 4): every off-diagonal cell, two pairs exchanging at a time;
each plain (st.relaxed.sys / ld.acquire.sys, the barrier's signal when nothing was published) and fenced (fence.sys
before every store, the signal after a publication).  Every cell's digest is checked by the library (status 0).
This is signal latency through L2 over a VMM mapping of the same HBM, not NVLink, which needs two GPUs and is not
measured here.  Prints one JSON document with the card's name, power limit and SM clock read in the same call
(read-only query)."""
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
ap.add_argument("--trips", type=int, default=1024)
ap.add_argument("--reps", type=int, default=32)
ap.add_argument("--out", default=None, help="also write the JSON document to this file")
a = ap.parse_args()


def gpu():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def cells(pp):
    out = {}
    for i in range(pp.n):
        for j in range(pp.n):
            if i == j:
                continue
            assert pp.measured[i][j] and pp.status[i][j] == 0, (i, j, pp.status[i][j])
            out[f"cell_{i}_{j}"] = {"ns_min": pp.ns_min[i][j], "ns_median": pp.ns_median[i][j], "ns_max": pp.ns_max[i][j]}
    med = [c["ns_median"] for c in out.values()]
    return {"median_of_cell_medians": statistics.median(med), "min_cell_median": min(med), "max_cell_median": max(med),
            **out}


res = {"trips": a.trips, "reps": a.reps,
       "what": "ns per signal round trip (st.relaxed.sys store into the peer's line, ld.acquire.sys poll of the local "
               "line, both ways) between ranks sharing one GPU through VMM mappings of its HBM; one untimed warm-up "
               "rep first; fenced: __threadfence_system (MEMBAR.SC.SYS) before every store"}
SAME = pkg.abi.FLAG_ALLOW_SAME_DEVICE | pkg.abi.FLAG_NO_COOPERATIVE
for n in (2, 4):
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=1 << 20, flags=SAME, ctas=8, timeout_ms=20000)) as p:
        for fenced in (False, True):
            pp = p.PingPong(a.trips, a.reps, fenced)
            res[f"n{n}_same_device_{'fenced' if fenced else 'plain'}"] = {**cells(pp), "call_ms": pp.ms}
res["gpu"] = gpu()
res["nvlink"] = "not measured (one GPU)"
if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
print(json.dumps(res, indent=1))
