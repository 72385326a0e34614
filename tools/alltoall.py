#!/usr/bin/env python3
"""The one-shot all-to-all of cdprobe_alltoall on one GPU, per rank and size: ns per rep (min / median / max over the
timed reps), the egress rate of the median (blocks x size / ns) and the summary t0_ns, peak_gbps and half_bytes:
  - one rank (N = 1) at `--bytes` on each write data path (TMA bulk, 16-byte and 32-byte ld/st).  The rank's one block
    is the loop-back block into its own exchange area, so the curve is a write curve of local HBM, and its t0_ns is
    the fixed cost of a write phase, next to the 6 us phase cost the default gate assumes;
  - two ranks on one device (`--pair-bytes`), each pushing one block to the other through a VMM mapping.
Every cell is checked word for word by the library (status 0).  NVLink needs two GPUs and is not measured here.
Prints a table, then one JSON document with the card's name, power limit and SM clock read in the same call (read-only
query); --out also writes the document to a file."""
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
ap.add_argument("--pair-bytes", type=int, default=256 << 20)
ap.add_argument("--reps", type=int, default=16)
ap.add_argument("--out", default=None, help="also write the JSON document to this file")
a = ap.parse_args()
PHASE_OVERHEAD_NS = 6000.0  # the default gate's fixed phase cost (handle.cc kPhaseOverheadNs)


def gpu():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def rows(aa):
    for s in range(aa.n):
        for d in range(aa.n):
            if aa.cell_measured[s][d]:
                assert aa.cell_status[s][d] == 0 and aa.bad_sizes[s][d] == 0, (s, d, aa.cell_status[s][d])
    out = {}
    for r in range(aa.n):
        assert aa.measured[r] and aa.status[r] == 0, (r, aa.status[r])
        b = aa.blocks[r]
        out[f"rank_{r}"] = {
            "blocks": b, "t0_ns": aa.t0_ns[r], "peak_gbps": aa.peak_gbps[r], "half_bytes": aa.half_bytes[r],
            "sizes": [{"bytes": s, "ns_min": lo, "ns_median": med, "ns_max": hi, "egress_gbps_median": b * s / med}
                      for s, lo, med, hi in zip(aa.sizes, aa.ns_min[r], aa.ns_median[r], aa.ns_max[r])]}
    return out


res = {"bytes": a.bytes, "pair_bytes": a.pair_bytes, "reps": a.reps, "gate_phase_overhead_ns": PHASE_OVERHEAD_NS,
       "what": "ns per rep of the one-shot all-to-all: every rank pushes the first `bytes` of a block to every cell it "
               "has, interleaved, with its whole probe grid on the probe's write data path, from the rep's barrier "
               "release stamp to the rank's last CTA completion stamp after its stores and a fence.sys (%globaltimer); "
               "one untimed warm-up rep per size first; egress_gbps_median = blocks x bytes / ns_median"}
for path, name in enumerate(("tma", "ldst16", "ldst32")):
    with pkg.Open(pkg.Config(ordinals=[0], bytes=a.bytes, timeout_ms=20000)) as p:
        p.SetOption(pkg.abi.OPT_PATH, path)
        aa = p.AllToAll(a.reps)
        res[f"n1_{name}"] = {**rows(aa), "call_ms": aa.ms}
with pkg.Open(pkg.Config(ordinals=[0, 0], bytes=a.pair_bytes, flags=0x40 | 0x10, ctas=66, timeout_ms=20000)) as p:
    aa = p.AllToAll(a.reps)
    res["n2_same_device_tma"] = {**rows(aa), "call_ms": aa.ms}
res["gpu"] = gpu()
res["nvlink"] = "not measured (one GPU)"

print(f"{'run':10} {'bytes':>12} {'ns_min':>12} {'ns_median':>12} {'ns_max':>12} {'egress GB/s':>12}")
for name in ("n1_tma", "n1_ldst16", "n1_ldst32", "n2_same_device_tma"):
    for s in res[name]["rank_0"]["sizes"]:
        print(f"{name:10} {s['bytes']:12d} {s['ns_min']:12.0f} {s['ns_median']:12.0f} {s['ns_max']:12.0f} "
              f"{s['egress_gbps_median']:12.1f}")
for name in ("n1_tma", "n1_ldst16", "n1_ldst32"):
    print(f"{name}: write t0_ns {res[name]['rank_0']['t0_ns']:.0f} against the gate's {PHASE_OVERHEAD_NS:.0f}")
print(f"gpu: {res['gpu']}")
if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
print(json.dumps(res))
