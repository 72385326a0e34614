#!/usr/bin/env python3
"""Bandwidth versus transfer size of cdprobe_bwcurve on one GPU, per cell and size: ns per rep (min / median / max over
the timed reps) and GB/s of the median, with the summary t0_ns, peak_gbps and half_bytes:
  - one rank (N = 1) at 1 GiB: the loop-back cell on each read data path (TMA bulk, 16-byte and 32-byte ld/st);
  - two ranks on the same device (N = 2), 1 GiB sliced, TMA path, 64 CTAs each so both grids fit the SMs at once:
    both cells of the pair read at the same time.
Every cell's checksums are checked by the library (status 0).  On one device the reads are served by the same HBM and
L2: sizes up to the 50 MB L2 come from L2 after the warm-up rep, larger ones from HBM.  NVLink needs two GPUs and is
not measured here.  Prints one JSON document with the card's name, power limit and SM clock read in the same call
(read-only query)."""
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
ap.add_argument("--bytes", type=int, default=1 << 30)
ap.add_argument("--reps", type=int, default=16)
ap.add_argument("--out", default=None, help="also write the JSON document to this file")
a = ap.parse_args()


def gpu():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def cells(bw):
    out = {}
    for i in range(bw.n):
        for j in range(bw.n):
            if i == j and bw.n > 1:
                continue
            assert bw.measured[i][j] and bw.status[i][j] == 0 and bw.bad_sizes[i][j] == 0, (i, j, bw.status[i][j])
            out[f"cell_{i}_{j}"] = {
                "t0_ns": bw.t0_ns[i][j], "peak_gbps": bw.peak_gbps[i][j], "half_bytes": bw.half_bytes[i][j],
                "sizes": [{"bytes": s, "ns_min": lo, "ns_median": med, "ns_max": hi, "gbps_median": s / med}
                          for s, lo, med, hi in zip(bw.sizes, bw.ns_min[i][j], bw.ns_median[i][j], bw.ns_max[i][j])]}
    return out


res = {"bytes": a.bytes, "reps": a.reps,
       "what": "ns per rep of reading the first `bytes` of the cell's source slice with the rank's whole probe grid "
               "(one CTA per SM, every CTA reading) on the probe's read data path, from a grid barrier's release "
               "stamp to the last CTA's completion stamp (%globaltimer); one untimed warm-up rep per size first; "
               "gbps_median = bytes / ns_median"}
for path, name in enumerate(("tma", "ldst16", "ldst32")):
    with pkg.Open(pkg.Config(ordinals=[0], bytes=a.bytes, timeout_ms=20000)) as p:
        p.SetOption(pkg.abi.OPT_PATH, path)
        bw = p.BwCurve(a.reps)
        res[f"n1_loopback_{name}"] = {**cells(bw), "call_ms": bw.ms}
SAME = pkg.abi.FLAG_ALLOW_SAME_DEVICE | pkg.abi.FLAG_NO_COOPERATIVE
with pkg.Open(pkg.Config(ordinals=[0, 0], bytes=a.bytes, flags=SAME, ctas=64, timeout_ms=20000)) as p:
    bw = p.BwCurve(a.reps)
    res["n2_same_device_tma"] = {**cells(bw), "call_ms": bw.ms}
res["gpu"] = gpu()
res["nvlink"] = "not measured (one GPU)"
if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
print(json.dumps(res))
