#!/usr/bin/env python3
"""Remote atomics of cdprobe_atomics on one GPU, ns per atomic (min / median / max over the timed reps):
  - one rank (N = 1): the loop-back cell, local L2 atomics through the VMM mapping;
  - two and four ranks on the same device (N = 2, 4): every off-diagonal cell, all issuers at once;
each for every kind: a dependent fetch-add chain, a dependent CAS chain (one lane each), and 32 lanes of one warp
running fetch-add chains on the same word (ns per atomic under 32-way contention).  Every cell's returns, read-back
and digest are checked by the library (status 0).  These are L2 atomics over VMM mappings of the same HBM, not NVLink,
which needs two GPUs and is not measured here.  Prints one JSON document with the card's name, power limit and SM
clock read in the same call (read-only query)."""
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
ap.add_argument("--ops", type=int, default=4096)
ap.add_argument("--reps", type=int, default=32)
ap.add_argument("--out", default=None, help="also write the JSON document to this file")
a = ap.parse_args()


def gpu():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def cells(at):
    out = {}
    for i in range(at.n):
        for j in range(at.n):
            if i == j and at.n > 1:
                continue
            assert at.measured[i][j] and at.status[i][j] == 0, (i, j, at.status[i][j])
            out[f"cell_{i}_{j}"] = {"ns_min": at.ns_min[i][j], "ns_median": at.ns_median[i][j],
                                    "ns_max": at.ns_max[i][j], "native": at.native[i][j]}
    med = [c["ns_median"] for c in out.values()]
    return {"median_of_cell_medians": statistics.median(med), "min_cell_median": min(med), "max_cell_median": max(med),
            **out}


res = {"ops": a.ops, "reps": a.reps,
       "what": "ns per system-scope 64-bit atomic (atom.relaxed.sys) on each cell's own word in the target's memory, "
               "issued through a VMM mapping of the same GPU's HBM; fetch_add / cas: one lane, each op's operand "
               "computed from the previous return; contended: 32 lanes of one warp on one word, ns per atomic = rep "
               "time / (32 x ops); one untimed warm-up rep first; several ranks run at once at N > 1"}
SAME = pkg.abi.FLAG_ALLOW_SAME_DEVICE | pkg.abi.FLAG_NO_COOPERATIVE
for n in (1, 2, 4):
    flags = 0 if n == 1 else SAME
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=1 << 20, flags=flags, ctas=8, timeout_ms=20000)) as p:
        for kind, name in enumerate(pkg.abi.ATOMIC_KIND_NAMES):
            at = p.Atomics(kind, a.ops, a.reps)
            res[f"n{n}_{'loopback' if n == 1 else 'same_device'}_{name}"] = {**cells(at), "call_ms": at.ms}
res["gpu"] = gpu()
res["nvlink"] = "not measured (one GPU)"
if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
print(json.dumps(res, indent=1))
