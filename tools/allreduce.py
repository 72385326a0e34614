#!/usr/bin/env python3
"""The one-shot all-reduce of cdprobe_allreduce on one GPU, per rank and size: ns per rep (min / median / max over the
timed reps), the algorithm bandwidth of the median (size / ns) and the summary t0_ns, peak_gbps and half_bytes:
  - one rank (N = 1) at `--bytes` on each read data path (TMA bulk, 16-byte and 32-byte ld/st).  The output is a copy
    of the rank's own prefix, so a rep moves 2 x size through HBM: size read, size written.
Every row's checksums and words are checked by the library (status 0).  Sizes up to the 50 MB L2 come from L2 after
the warm-up rep, larger ones from HBM.  With N ranks each rank's NVLink ingress is (n - 1) x the algorithm bandwidth;
NVLink needs two GPUs and is not measured here.  Prints a table, then one JSON document with the card's name, power
limit and SM clock read in the same call (read-only query); --out also writes the document to a file."""
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


def rows(ar):
    out = {}
    for r in range(ar.n):
        assert ar.measured[r] and ar.status[r] == 0 and ar.bad_sizes[r] == 0, (r, ar.status[r])
        assert all(b == 0 for b in ar.bad_words[r]), r
        out[f"rank_{r}"] = {
            "t0_ns": ar.t0_ns[r], "peak_gbps": ar.peak_gbps[r], "half_bytes": ar.half_bytes[r],
            "sizes": [{"bytes": s, "ns_min": lo, "ns_median": med, "ns_max": hi, "algbw_gbps_median": s / med}
                      for s, lo, med, hi in zip(ar.sizes, ar.ns_min[r], ar.ns_median[r], ar.ns_max[r])]}
    return out


res = {"bytes": a.bytes, "reps": a.reps,
       "what": "ns per rep of the one-shot all-reduce of the first `bytes` of every rank's source buffer into the "
               "rank's own memory, with the rank's whole probe grid (one CTA per SM) on the probe's read data path, "
               "from the rep's barrier release stamp to the rank's last CTA completion stamp (%globaltimer); one "
               "untimed warm-up rep per size first; algbw_gbps_median = bytes / ns_median (bytes per ns)"}
for path, name in enumerate(("tma", "ldst16", "ldst32")):
    with pkg.Open(pkg.Config(ordinals=[0], bytes=a.bytes, timeout_ms=20000)) as p:
        p.SetOption(pkg.abi.OPT_PATH, path)
        ar = p.AllReduce(a.reps)
        res[f"n1_{name}"] = {**rows(ar), "call_ms": ar.ms}
res["gpu"] = gpu()
res["nvlink"] = "not measured (one GPU)"

print(f"{'path':8} {'bytes':>12} {'ns_min':>12} {'ns_median':>12} {'ns_max':>12} {'algbw GB/s':>11}")
for name in ("tma", "ldst16", "ldst32"):
    for s in res[f"n1_{name}"]["rank_0"]["sizes"]:
        print(f"{name:8} {s['bytes']:12d} {s['ns_min']:12.0f} {s['ns_median']:12.0f} {s['ns_max']:12.0f} "
              f"{s['algbw_gbps_median']:11.1f}")
print(f"gpu: {res['gpu']}")
if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
print(json.dumps(res))
