#!/usr/bin/env python3
"""Copy-engine bandwidth versus transfer size of cdprobe_memcpy on one GPU, pulled (OP_READ) and pushed (OP_WRITE), with
cdprobe_bwcurve's SM read curve of the same handle beside it:
  - one rank (N = 1) at 4 MiB and at 1 GiB: the loop-back cell, a device-to-device copy within local HBM;
  - N = 2, 4 and 8 ranks on the same device, 256 MiB sliced: the cells of a round copy at once, each rank on its own
    stream, so they share the device's copy engines and HBM.
Every cell's words are checked by the library (status 0, no bad word).  Per cell and size: ns per copy (min / median /
max over the timed reps, by CUDA events, which resolve about 0.5 us) and GB/s of the median, with the summary t0_ns,
peak_gbps and half_bytes.  NVLink needs two GPUs and is not measured here.  Writes one JSON document with the card's
name, power limit and SM clock read in the same call (read-only query)."""
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
ap.add_argument("--reps", type=int, default=8)
ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_memcpy_n1.json"))
a = ap.parse_args()
SAME = pkg.abi.FLAG_ALLOW_SAME_DEVICE | pkg.abi.FLAG_NO_COOPERATIVE


def gpu():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def cells(m, checked):
    out = {}
    for i in range(m.n):
        for j in range(m.n):
            if i == j and m.n > 1:
                continue
            assert m.measured[i][j] and m.status[i][j] == 0 and m.bad_sizes[i][j] == 0, (i, j, m.status[i][j])
            if checked:
                assert m.bad_words[i][j] == [0] * len(m.sizes), (i, j)
            out[f"cell_{i}_{j}"] = {
                "t0_ns": m.t0_ns[i][j], "peak_gbps": m.peak_gbps[i][j], "half_bytes": m.half_bytes[i][j],
                "ns_min": m.ns_min[i][j], "ns_median": m.ns_median[i][j], "ns_max": m.ns_max[i][j],
                "gbps_median": [round(s / med, 2) for s, med in zip(m.sizes, m.ns_median[i][j])]}
    return out


def measure(n, nbytes):
    cfg = pkg.Config(ordinals=[0] * n, bytes=nbytes, timeout_ms=30000,
                     **({} if n == 1 else dict(flags=SAME, ctas=128 // n)))
    res = {}
    with pkg.Open(cfg) as p:
        for op, name in ((pkg.abi.OP_READ, "pull"), (pkg.abi.OP_WRITE, "push")):
            m = p.Memcpy(op, a.reps)
            res[f"memcpy_{name}"] = {"sizes": m.sizes, **cells(m, True), "call_ms": m.ms, "area_bytes": m.area_bytes}
        bw = p.BwCurve(a.reps)
        res["bwcurve_sm_read"] = {"sizes": bw.sizes, **cells(bw, False), "call_ms": bw.ms, "path": bw.path}
    return res


res = {"reps": a.reps,
       "what": "memcpy_*: ns per cudaMemcpyAsync of the first `bytes` of the cell's source slice on the issuer's "
               "stream, from the event after a stream wait the host releases once the rep is queued to the event "
               "after the copy; pull = target's slice into the issuer's exchange area, push = issuer's slice into the "
               "target's; one untimed warm-up rep per size first; every landed word checked after each rep. "
               "bwcurve_sm_read: the same handle's cdprobe_bwcurve (SM loads, %globaltimer). Per cell, lists over "
               "`sizes`; gbps_median = size / ns_median",
       "n1_4MiB": measure(1, 4 << 20), "n1_1GiB": measure(1, 1 << 30)}
for n in (2, 4, 8):
    res[f"n{n}_same_device_256MiB"] = measure(n, 256 << 20)
res["gpu"] = gpu()
res["nvlink"] = "not measured (one GPU)"
os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
with open(a.out, "w") as f:
    json.dump(res, f)
for k, v in res.items():
    if k.startswith("n") and isinstance(v, dict):
        print(k, {kind: max(c["peak_gbps"] for name, c in cs.items() if name.startswith("cell_"))
                  for kind, cs in v.items()})
print("gpu", res["gpu"])
