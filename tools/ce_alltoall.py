#!/usr/bin/env python3
"""The copy-engine all-to-all of cdprobe_ce_alltoall on one GPU, pulled (OP_READ) and pushed (OP_WRITE), with
cdprobe_alltoall (the same traffic on the SMs) and cdprobe_memcpy (the same cells, one round at a time) of the same
handle beside it:
  - one rank (N = 1) at 256 MiB: the loop-back block only;
  - N = 2, 4 and 8 ranks sharing the device, 256 MiB sliced: every block of the domain copied at once, each on a copy
    stream of its own, the ranks signalling each other with stream memory operations.
A domain whose streams exceed the default 8 hardware queues runs in child processes with CUDA_DEVICE_MAX_CONNECTIONS=32,
as many as keep each within 32 (N = 8: two processes of four ranks).
Every block's words are checked by the library.  Per rank and size: ns per rep (median over the timed reps, from the
release until every block addressed to the rank has landed) and blocks x size / ns; per cell, the median copy time.
NVLink, stream writes through another GPU's mapping, the stream-signal latency between GPUs and how many copy engines a
GPU drives at once need several GPUs and are not measured here.  Writes one JSON document with the card's name, power
limit and SM clock read in the same call (read-only query)."""
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
ap.add_argument("--bytes", type=int, default=256 << 20)
ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_ce_alltoall_n1.json"))
ap.add_argument("--one", type=int, default=0, help="measure this rank count only and print its JSON (child process)")
ap.add_argument("--world", type=int, default=1)
ap.add_argument("--rank", type=int, default=0)
ap.add_argument("--session", default="")
a = ap.parse_args()
SAME = pkg.abi.FLAG_ALLOW_SAME_DEVICE | pkg.abi.FLAG_NO_COOPERATIVE


def gpu():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def rate(sizes, ns, blocks=1):
    return [round(blocks * s / t, 2) if t else None for s, t in zip(sizes, ns)]


def ce(m):
    rows = {}
    for r in range(m.n):
        if not m.row_mask >> r & 1:
            continue
        assert m.measured[r] and m.status[r] == 0, (r, m.status[r])
        rows[f"rank_{r}"] = {"blocks": m.blocks[r], "ns_median": m.ns_median[r], "ns_max": m.ns_max[r],
                             "gbps_median": rate(m.sizes, m.ns_median[r], m.blocks[r]), "peak_gbps": m.peak_gbps[r],
                             "copy_ns_median": {str(j): m.copy_ns_median[r][j] for j in range(m.n)
                                                if m.copy_ns_median[r][j] is not None}}
    for s in range(m.n):
        for d in range(m.n):
            if m.cell_measured[s][d]:
                assert m.cell_status[s][d] == 0 and m.bad_words[s][d] == [0] * len(m.sizes), (s, d)
    return {"sizes": m.sizes, "call_ms": m.ms, **rows}


def measure(n):
    n_local = n // a.world
    mine = range(a.rank * n_local, (a.rank + 1) * n_local)
    cfg = pkg.Config(ordinals=[0] * n_local, bytes=a.bytes, timeout_ms=30000, world_size=a.world, rank=a.rank,
                     session=a.session, **({} if n == 1 else dict(flags=SAME, ctas=128 // n)))
    res = {"n": n, "gpu": gpu(), "max_connections": os.environ.get("CUDA_DEVICE_MAX_CONNECTIONS", "8 (default)")}
    with pkg.Open(cfg) as p:
        for op, name in ((pkg.abi.OP_READ, "pull"), (pkg.abi.OP_WRITE, "push")):
            res[f"ce_alltoall_{name}"] = ce(p.CeAllToAll(op, a.reps))
        aa = p.AllToAll(a.reps)
        assert all(aa.cell_status[s][d] == 0 for s in range(n) for d in mine if s != d or n == 1)
        res["alltoall"] = {"sizes": aa.sizes, "call_ms": aa.ms, **{
            f"rank_{r}": {"blocks": aa.blocks[r], "ns_median": aa.ns_median[r], "peak_gbps": aa.peak_gbps[r],
                          "gbps_median": rate(aa.sizes, aa.ns_median[r], aa.blocks[r])} for r in mine}}
        for op, name in ((pkg.abi.OP_READ, "pull"), (pkg.abi.OP_WRITE, "push")):
            m = p.Memcpy(op, a.reps)
            res[f"memcpy_{name}"] = {"sizes": m.sizes, "call_ms": m.ms, **{
                f"cell_{i}_{j}": {"ns_median": m.ns_median[i][j], "peak_gbps": m.peak_gbps[i][j]}
                for i in range(n) for j in range(n) if m.measured[i][j] and m.status[i][j] == 0}}
    return res


if a.one:
    print("RESULT " + json.dumps(measure(a.one)))
    sys.exit(0)

doc = {"tool": "tools/ce_alltoall.py", "reps": a.reps, "bytes": a.bytes, "runs": []}
for n in (1, 2, 4, 8):
    # each rank holds its own stream and one copy stream per block it copies: n streams (the loop-back adds one at
    # N = 1) per rank, at most 8 per device by default and 32 with the variable set
    per_rank = n + (1 if n == 1 else 0)
    world = 1
    while (n // world) * per_rank > 32:
        world *= 2
    env = dict(os.environ, **({"CUDA_DEVICE_MAX_CONNECTIONS": "32"} if (n // world) * per_rank > 8 else {}))
    session = f"ce-a2a-{os.getpid()}-{n}"
    procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), "--one", str(n), "--reps", str(a.reps),
                               "--bytes", str(a.bytes), "--world", str(world), "--rank", str(r), "--session", session],
                              env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for r in range(world)]
    parts = []
    for pr in procs:
        so, se = pr.communicate(timeout=1800)
        assert pr.returncode == 0, se[-4000:]
        parts.append(json.loads([l for l in so.splitlines() if l.startswith("RESULT ")][-1][7:]))
    run = parts[0]
    for part in parts[1:]:  # every process adds its own ranks' rows and cells
        for key, val in part.items():
            if isinstance(val, dict) and key != "gpu":
                run[key].update({k: v for k, v in val.items() if k.startswith(("rank_", "cell_"))})
    run["processes"] = world
    doc["runs"].append(run)
    pull, push = run["ce_alltoall_pull"], run["ce_alltoall_push"]
    print(f"N={n}: pull peak {max(pull[f'rank_{r}']['peak_gbps'] for r in range(n)):.1f} GB/s per rank, "
          f"push {max(push[f'rank_{r}']['peak_gbps'] for r in range(n)):.1f}; "
          f"SM all-to-all {max(run['alltoall'][f'rank_{r}']['peak_gbps'] for r in range(n)):.1f}")
os.makedirs(os.path.dirname(a.out), exist_ok=True)
with open(a.out, "w") as f:
    json.dump(doc, f, indent=1)
print("wrote", a.out)
