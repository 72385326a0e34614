#!/usr/bin/env python3
"""Tuning sweep on the GPU box: path x CTA count (x N in-process GPUs). Writes JSON lines."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cdprobe_pkg  # noqa: E402

pkg = cdprobe_pkg.load()
abi = pkg.abi

ap = argparse.ArgumentParser()
ap.add_argument("--gpus", type=int, default=1)
ap.add_argument("--bytes", type=int, default=1 << 30)
ap.add_argument("--mode", default="sliced")
ap.add_argument("--ctas", default="132,128,96,66,64,48,32")
ap.add_argument("--iters", type=int, default=8)
ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "sweep.jsonl"))
ap.add_argument("--overlap", default="0")
ap.add_argument("--uni", default="0")
ap.add_argument("--paths", default="0,1")
ap.add_argument("--vctas", type=int, default=32)
ap.add_argument("--barriers", default="0", help="0 = default (neighbourhood + no wait write->read), 1 = all-rank (round 1), "
                                              "2 = neighbourhood with the pair exchange kept between write and read")
args = ap.parse_args()

mode = {"sliced": 1, "full": 2, "reach": 0}[args.mode]
n = args.gpus
os.makedirs(os.path.dirname(args.out), exist_ok=True)
with pkg.Open(pkg.Config(ordinals=list(range(n)), bytes=args.bytes, mode=mode, timeout_ms=20000)) as p, open(args.out, "a") as f:
    p.SetOption(abi.OPT_EVENT_TIMING, 1)
    p.SetOption(abi.OPT_VERIFY_CTAS, args.vctas)
    for uni, overlap in [(int(u), int(x)) for u in args.uni.split(",") for x in args.overlap.split(",")]:
        p.SetOption(abi.OPT_UNIDIRECTIONAL, uni)
        p.SetOption(abi.OPT_OVERLAP_VERIFY, overlap)
        for allrank in [int(b) for b in args.barriers.split(",")]:
            p.SetOption(abi.OPT_ALL_RANK_BARRIERS, 1 if allrank == 1 else 0)
            p.SetOption(abi.OPT_PAIR_BARRIERS, 1 if allrank == 2 else 0)
            for path in [int(x) for x in args.paths.split(",")]:
                p.SetOption(abi.OPT_PATH, path)
                for ctas in [int(c) for c in args.ctas.split(",")]:
                    p.SetOption(abi.OPT_CTAS, ctas)
                    for _ in range(2):
                        p.Run()
                    rs = [p.Run() for _ in range(args.iters)]
                    off = [(i, j) for i in range(n) for j in range(n) if i != j or n == 1]
                    rec = {
                        "n": n, "mode": args.mode, "bytes": args.bytes, "path": ("tma", "ldst", "ldst256")[path], "ctas": ctas,
                        "overlap": overlap, "uni": uni, "all_rank_barriers": allrank, "bpp": rs[0].bytes_per_pair, "phases": rs[0].phases,
                        "probe_ms": statistics.median(r.probe_ms for r in rs),
                        "probe_ms_min": min(r.probe_ms for r in rs),
                        "event_ms": statistics.median(max(r.event_ms) for r in rs),
                        "device_ms": statistics.median(max(r.device_ms) for r in rs),
                        "barrier_us": statistics.median(max(r.barrier_us) for r in rs),
                        "read_min": statistics.median(min(r.gbps_read[i][j] for i, j in off) for r in rs),
                        "read_max": statistics.median(max(r.gbps_read[i][j] for i, j in off) for r in rs),
                        "write_min": statistics.median(min(r.gbps_write[i][j] for i, j in off) for r in rs),
                        "write_max": statistics.median(max(r.gbps_write[i][j] for i, j in off) for r in rs),
                        "verdict": all(r.verdict for r in rs),
                        "reach": all(all(all(c == 1 for c in row) for row in r.reach) for r in rs),
                    }
                    f.write(json.dumps(rec) + "\n")
                    f.flush()
                    print(json.dumps(rec))
