#!/usr/bin/env python3
"""The one-shot all-reduce of cdprobe_allreduce on one GPU, per rank and size: ns per rep (min / median / max over the
timed reps), the algorithm bandwidth of the median (size / ns) and the summary t0_ns, peak_gbps and half_bytes:
  - one rank (N = 1) at `--bytes` on each read data path (TMA bulk, 16-byte and 32-byte ld/st).  The output is a copy
    of the rank's own prefix, so a rep moves 2 x size through HBM: size read, size written.
Every row's checksums and words are checked by the library (status 0).  Sizes up to the 50 MB L2 come from L2 after
the warm-up rep, larger ones from HBM.  With N ranks each rank's NVLink ingress is (n - 1) x the algorithm bandwidth;
NVLink needs two GPUs and is not measured here.  Prints a table, then one JSON document with the card's name, power
limit and SM clock read in the same call (read-only query); --out also writes the document to a file.

--twoshot adds cdprobe_allreduce_twoshot in the same session: at N = 1 on each path next to the one-shot (the rank owns
every unit, so a rep is the one-shot's reads plus a store to its own gather area and the untimed check), and with 2 and
4 ranks sharing GPU 0 (`--multi-bytes` per rank) on the TMA path.  Each rank's link traffic in a two-shot rep is
2 (n - 1) / n x size, so its bus bandwidth, busbw = algbw x 2 (n - 1) / n, is the figure nccl-tests reports; ranks on
one device move that traffic through its own HBM, not NVLink.

--ll measures cdprobe_allreduce_ll instead, next to the one-shot and the two-shot (TMA path) on the same handle in the
same session: N = 1 and 2, 4 and 8 ranks sharing GPU 0 at `--ll-bytes` per pair (default 1 MiB, the LL ladder's
largest size), so the ladder runs 4 KiB ... 1 MiB.  An LL rep runs from the end of the rank's previous rep to the end of
its own (no barrier per rep); a one-shot rep from its opening barrier's release, a two-shot rep to its closing
release.  Each rank's link ingress per LL rep is 2 (n - 1) x size: every 8 bytes of data travel in a 16-byte packet.

--ring measures cdprobe_allreduce_ring instead, next to the one-shot and the two-shot (TMA path) on the same handle in
the same session: N = 1 at `--bytes` per pair, and 2, 4 and 8 ranks sharing GPU 0 at `--multi-bytes` per pair.  A ring
rep runs from its opening barrier's release to the moment the rank's output is complete.  Each rank sends and receives
2 (n - 1) / n x size per ring rep, over one link each, so busbw = algbw x 2 (n - 1) / n is reported for all three.

--push measures cdprobe_allreduce_push instead, next to the one-shot and the two-shot on the same handle in the same
session: N = 1 at `--bytes` per pair on each data path (TMA bulk reductions, and red.global per word behind 16-byte and
32-byte loads), and 2, 4 and 8 ranks sharing GPU 0 at `--multi-bytes` per pair on the TMA path.  A push rep runs from
its opening barrier's release to its closing release, as a two-shot rep does.  Each rank's link traffic per rep is the
two-shot's, 2 (n - 1) / n x size, every transfer a write, so busbw = algbw x 2 (n - 1) / n is reported for all three.

--nvls measures cdprobe_allreduce_nvls instead, next to the one-shot and the two-shot (TMA path) on the same handle in
the same session, one rank per visible device (up to 8) at `--bytes` per pair.  It records in the same call the
device's CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, the VMM and multicast minimum granularities, the CUresult of a
direct cuMulticastCreate of a one-device object, and the card's name, power limit and SM clock.  Where the NVLS call
runs nothing (a driver that refuses a one-device object, on one GPU), its rows' status and cdprobe_last_error are
recorded next to the one-shot's and the two-shot's times."""
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
ap.add_argument("--twoshot", action="store_true", help="also measure cdprobe_allreduce_twoshot")
ap.add_argument("--multi-bytes", type=int, default=256 << 20, help="bytes_per_pair of the 2- and 4-rank two-shot runs")
ap.add_argument("--ll", action="store_true", help="measure cdprobe_allreduce_ll next to the one-shot and the two-shot")
ap.add_argument("--ll-bytes", type=int, default=1 << 20, help="bytes_per_pair of the --ll runs")
ap.add_argument("--ring", action="store_true", help="measure cdprobe_allreduce_ring next to the one-shot and two-shot")
ap.add_argument("--push", action="store_true", help="measure cdprobe_allreduce_push next to the one-shot and two-shot")
ap.add_argument("--nvls", action="store_true", help="measure cdprobe_allreduce_nvls next to the one-shot and two-shot")
a = ap.parse_args()


def gpu():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))


def rows(ar, bus=None):
    """Per rank: the summary and every size; bus: also busbw_gbps_median = algbw x bus."""
    out = {}
    for r in range(ar.n):
        assert ar.measured[r] and ar.status[r] == 0 and ar.bad_sizes[r] == 0, (r, ar.status[r])
        assert all(b == 0 for b in ar.bad_words[r]), r
        out[f"rank_{r}"] = {
            "t0_ns": ar.t0_ns[r], "peak_gbps": ar.peak_gbps[r], "half_bytes": ar.half_bytes[r],
            "sizes": [{"bytes": s, "ns_min": lo, "ns_median": med, "ns_max": hi, "algbw_gbps_median": s / med,
                       **({} if bus is None else {"busbw_gbps_median": s / med * bus})}
                      for s, lo, med, hi in zip(ar.sizes, ar.ns_min[r], ar.ns_median[r], ar.ns_max[r])]}
        if bus is not None:
            out[f"rank_{r}"]["peak_busbw_gbps"] = ar.peak_gbps[r] * bus
    return out


def multicast_facts():
    """CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED of device 0, the minimum VMM and multicast granularities for a
    one-device object of 2 MiB, and the CUresult of cuMulticastCreate for such an object (POSIX fd handle type; 0:
    created, and released at once), read through the driver API on device 0's primary context."""
    import ctypes as C

    class McProp(C.Structure):
        _fields_ = [("numDevices", C.c_uint), ("size", C.c_size_t), ("handleTypes", C.c_ulonglong),
                    ("flags", C.c_ulonglong)]

    class Loc(C.Structure):
        _fields_ = [("type", C.c_int), ("id", C.c_int)]

    class AllocProp(C.Structure):
        _fields_ = [("type", C.c_int), ("requestedHandleTypes", C.c_int), ("location", Loc), ("win32HandleMetaData",
                    C.c_void_p), ("compressionType", C.c_ubyte), ("gpuDirectRDMACapable", C.c_ubyte),
                    ("usage", C.c_ushort), ("reserved", C.c_ubyte * 4)]

    cu = C.CDLL("libcuda.so.1")
    dev, on, mc, vmm = C.c_int(), C.c_int(), C.c_size_t(), C.c_size_t()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(C.byref(dev), 0) == 0
    assert cu.cuDeviceGetAttribute(C.byref(on), 132, dev) == 0  # CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED
    ap_ = AllocProp(1, 0, Loc(1, dev.value))  # pinned, on device 0
    assert cu.cuMemGetAllocationGranularity(C.byref(vmm), C.byref(ap_), 0) == 0
    rc = cu.cuMulticastGetGranularity(C.byref(mc), C.byref(McProp(1, 2 << 20, 0, 0)), 0)
    ctx, obj, name = C.c_void_p(), C.c_ulonglong(), C.c_char_p()
    assert cu.cuDevicePrimaryCtxRetain(C.byref(ctx), dev) == 0 and cu.cuCtxPushCurrent(ctx) == 0
    created = cu.cuMulticastCreate(C.byref(obj), C.byref(McProp(1, 2 << 20, 1, 0)))  # 1: POSIX file descriptor
    if created == 0:
        cu.cuMemRelease(obj)
    cu.cuGetErrorName(created, C.byref(name))
    cu.cuCtxPopCurrent(C.byref(C.c_void_p()))
    cu.cuDevicePrimaryCtxRelease(dev)
    return {"multicast_supported": on.value, "vmm_granularity_min": vmm.value,
            "multicast_granularity_min": mc.value if rc == 0 else f"CUresult {rc}",
            "create_one_device_2mib": {"curesult": created, "name": name.value.decode() if name.value else None}}


if a.nvls:
    import torch

    n_dev = torch.cuda.device_count()
    res = {"bytes": a.bytes, "reps": a.reps, "devices": n_dev, "multicast": multicast_facts(),
           "what": "cdprobe_allreduce_nvls (nvls), cdprobe_allreduce (one_shot) and cdprobe_allreduce_twoshot "
                   "(two_shot, TMA path) called one after another on the same handle, one rank per visible device "
                   "(N = 1 on one GPU) with one CTA per SM and bytes per pair: ns per rep of every size of the bwcurve "
                   "ladder for every call that ran, and the NVLS call's per-rank status where it ran nothing.  An nvls "
                   "or two-shot rep runs from its opening to its closing barrier release; a one-shot rep from its "
                   "opening barrier release to its latest CTA stamp.  algbw_gbps_median = bytes / ns_median; "
                   "busbw_gbps_median = algbw x 2 (n - 1) / n"}
    n = min(n_dev, 8)
    bus = 2 * (n - 1) / n
    with pkg.Open(pkg.Config(ordinals=list(range(n)), bytes=a.bytes * max(n - 1, 1), timeout_ms=60000)) as p:
        nvls = p.AllReduceNVLS(a.reps)
        nvls_error = p._lib.cdprobe_last_error().decode()
        one = p.AllReduce(a.reps)
        ts = p.AllReduceTwoShot(a.reps)
        ran = all(nvls.measured[r] for r in range(n))
        res[f"n{n}"] = {"nvls": {**(rows(nvls, bus) if ran else {"status": nvls.status, "last_error": nvls_error}),
                                 "call_ms": nvls.ms, "path": nvls.path},
                        "one_shot": {**rows(one, bus), "call_ms": one.ms},
                        "two_shot": {**rows(ts, bus), "call_ms": ts.ms}}
    res["gpu"] = gpu()
    res["nvlink"] = "not measured" if n == 1 else f"measured by the n{n} rows"
    runs = res[f"n{n}"]
    print(f"{'bytes':>11} {'nvls ns':>11} {'one-shot':>11} {'two-shot':>11}  (rank 0)")
    for i, (o, t) in enumerate(zip(runs["one_shot"]["rank_0"]["sizes"], runs["two_shot"]["rank_0"]["sizes"])):
        v = runs["nvls"]["rank_0"]["sizes"][i]["ns_median"] if ran else float("nan")
        print(f"{o['bytes']:11d} {v:11.0f} {o['ns_median']:11.0f} {t['ns_median']:11.0f}")
    print(f"nvls ran: {ran}  status: {nvls.status} {nvls_error}  multicast: {res['multicast']}  gpu: {res['gpu']}")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))
    sys.exit(0)

if a.push:
    res = {"bytes": a.bytes, "multi_bytes": a.multi_bytes, "reps": a.reps,
           "what": "ns per rep of cdprobe_allreduce_push (push), cdprobe_allreduce (one_shot) and "
                   "cdprobe_allreduce_twoshot (two_shot) called one after another on the same handle: n1_<path>: "
                   "N = 1 with one CTA per SM at bytes per pair on the tma, ldst16 and ldst32 data paths; n2, n4, n8: "
                   "2, 4, 8 ranks on GPU 0 (ALLOW_SAME_DEVICE | NO_COOPERATIVE, 16 CTAs each, TMA path) at "
                   "multi_bytes per pair; every size of the bwcurve ladder.  A push or two-shot rep runs from its "
                   "opening to its closing barrier release; a one-shot rep from its opening barrier release to its "
                   "latest CTA stamp.  algbw_gbps_median = bytes / ns_median; busbw_gbps_median = algbw x "
                   "2 (n - 1) / n"}
    runs = [(1, path) for path in (0, 1, 2)] + [(n, 0) for n in (2, 4, 8)]
    names = ("tma", "ldst16", "ldst32")
    for n, path in runs:
        bpp = a.bytes if n == 1 else a.multi_bytes
        cfg = pkg.Config(ordinals=[0] * n, bytes=bpp * max(n - 1, 1), flags=0x40 | 0x10 if n > 1 else 0,
                         ctas=16 if n > 1 else 0, timeout_ms=60000)
        bus = 2 * (n - 1) / n
        with pkg.Open(cfg) as p:
            p.SetOption(pkg.abi.OPT_PATH, path)
            push = p.AllReducePush(a.reps)
            one = p.AllReduce(a.reps)
            ts = p.AllReduceTwoShot(a.reps)
            res[f"n1_{names[path]}" if n == 1 else f"n{n}"] = {"push": {**rows(push, bus), "call_ms": push.ms},
                                                               "one_shot": {**rows(one, bus), "call_ms": one.ms},
                                                               "two_shot": {**rows(ts, bus), "call_ms": ts.ms}}
    res["gpu"] = gpu()
    res["nvlink"] = "not measured (one GPU)"
    print(f"{'run':>9} {'bytes':>11} {'push ns':>11} {'one-shot':>11} {'two-shot':>11} {'push algbw':>10} "
          f"{'push busbw':>10}  (rank 0)")
    for key in [f"n1_{x}" for x in names] + ["n2", "n4", "n8"]:
        for s, o, t in zip(*(res[key][x]["rank_0"]["sizes"] for x in ("push", "one_shot", "two_shot"))):
            print(f"{key:>9} {s['bytes']:11d} {s['ns_median']:11.0f} {o['ns_median']:11.0f} {t['ns_median']:11.0f} "
                  f"{s['algbw_gbps_median']:10.1f} {s['busbw_gbps_median']:10.1f}")
    print(f"gpu: {res['gpu']}")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))
    sys.exit(0)

if a.ring:
    res = {"bytes": a.bytes, "multi_bytes": a.multi_bytes, "reps": a.reps,
           "what": "ns per rep of cdprobe_allreduce_ring (ring), cdprobe_allreduce (one_shot) and "
                   "cdprobe_allreduce_twoshot (two_shot, TMA path) called one after another on the same handle: "
                   "N = 1 with one CTA per SM at bytes per pair, N = 2, 4, 8 ranks on GPU 0 (ALLOW_SAME_DEVICE | "
                   "NO_COOPERATIVE, 16 CTAs each) at multi_bytes per pair; every size of the bwcurve ladder.  A ring "
                   "rep runs from its opening barrier release to its latest CTA completion stamp; a one-shot rep from "
                   "its opening barrier release to its latest CTA stamp; a two-shot rep from its opening to its "
                   "closing barrier release.  algbw_gbps_median = bytes / ns_median; busbw_gbps_median = algbw x "
                   "2 (n - 1) / n"}
    for n in (1, 2, 4, 8):
        bpp = a.bytes if n == 1 else a.multi_bytes
        cfg = pkg.Config(ordinals=[0] * n, bytes=bpp * max(n - 1, 1), flags=0x40 | 0x10 if n > 1 else 0,
                         ctas=16 if n > 1 else 0, timeout_ms=60000)
        bus = 2 * (n - 1) / n
        with pkg.Open(cfg) as p:
            p.SetOption(pkg.abi.OPT_PATH, 0)
            ring = p.AllReduceRing(a.reps)
            one = p.AllReduce(a.reps)
            ts = p.AllReduceTwoShot(a.reps)
            res[f"n{n}"] = {"ring": {**rows(ring, bus), "call_ms": ring.ms},
                            "one_shot": {**rows(one, bus), "call_ms": one.ms},
                            "two_shot": {**rows(ts, bus), "call_ms": ts.ms}}
    res["gpu"] = gpu()
    res["nvlink"] = "not measured (one GPU)"
    print(f"{'n':>2} {'bytes':>11} {'ring ns':>11} {'one-shot':>11} {'two-shot':>11} {'ring algbw':>10} "
          f"{'ring busbw':>10}  (rank 0)")
    for n in (1, 2, 4, 8):
        for s, o, t in zip(*(res[f"n{n}"][x]["rank_0"]["sizes"] for x in ("ring", "one_shot", "two_shot"))):
            print(f"{n:2d} {s['bytes']:11d} {s['ns_median']:11.0f} {o['ns_median']:11.0f} {t['ns_median']:11.0f} "
                  f"{s['algbw_gbps_median']:10.1f} {s['busbw_gbps_median']:10.1f}")
    print(f"gpu: {res['gpu']}")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))
    sys.exit(0)

if a.ll:
    res = {"ll_bytes": a.ll_bytes, "reps": a.reps,
           "what": "ns per rep of cdprobe_allreduce_ll (ll), cdprobe_allreduce (one_shot) and "
                   "cdprobe_allreduce_twoshot (two_shot, TMA path) called one after another on the same handle: "
                   "N = 1 with one CTA per SM, N = 2, 4, 8 ranks on GPU 0 (ALLOW_SAME_DEVICE | NO_COOPERATIVE, 16 "
                   "CTAs each), bytes_per_pair = ll_bytes; the ll ladder is the bwcurve ladder up to 1 MiB and the "
                   "others are reported at the same sizes.  An ll rep runs from the end of the rank's previous rep "
                   "(the warm-up: its barrier release) to its latest CTA completion stamp; a one-shot rep from its "
                   "opening barrier release to its latest CTA stamp; a two-shot rep from its opening to its closing "
                   "barrier release.  algbw_gbps_median = bytes / ns_median; LL link ingress = 2 (n - 1) x bytes"}
    for n in (1, 2, 4, 8):
        cfg = pkg.Config(ordinals=[0] * n, bytes=a.ll_bytes * max(n - 1, 1), flags=0x40 | 0x10 if n > 1 else 0,
                         ctas=16 if n > 1 else 0, timeout_ms=20000)
        with pkg.Open(cfg) as p:
            ll = p.AllReduceLL(a.reps)
            one = p.AllReduce(a.reps)
            ts = p.AllReduceTwoShot(a.reps)
            res[f"n{n}"] = {"ll": {**rows(ll), "call_ms": ll.ms}, "one_shot": {**rows(one), "call_ms": one.ms},
                            "two_shot": {**rows(ts), "call_ms": ts.ms}}
    res["gpu"] = gpu()
    res["nvlink"] = "not measured (one GPU)"
    print(f"{'n':>2} {'rank':>4} {'bytes':>9} {'ll ns':>9} {'one-shot':>9} {'two-shot':>9} {'ll GB/s':>8}")
    for n in (1, 2, 4, 8):
        for r in range(n):
            rk = f"rank_{r}"
            for s, o, t in zip(*(res[f"n{n}"][x][rk]["sizes"] for x in ("ll", "one_shot", "two_shot"))):
                print(f"{n:2d} {r:4d} {s['bytes']:9d} {s['ns_median']:9.0f} {o['ns_median']:9.0f} "
                      f"{t['ns_median']:9.0f} {s['algbw_gbps_median']:8.1f}")
    print(f"gpu: {res['gpu']}")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))
    sys.exit(0)

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
        if a.twoshot:
            ts = p.AllReduceTwoShot(a.reps)
            res[f"twoshot_n1_{name}"] = {**rows(ts, 0.0), "call_ms": ts.ms}
if a.twoshot:
    res["twoshot_what"] = ("the same for the two-shot all-reduce (cdprobe_allreduce_twoshot): a rep runs from the "
                           "rank's opening domain-barrier release to its closing release, after every rank's pushes; "
                           "busbw_gbps_median = algbw x 2 (n - 1) / n.  twoshot_n2 / twoshot_n4: 2 and 4 ranks on "
                           "GPU 0 (ALLOW_SAME_DEVICE | NO_COOPERATIVE, 32 CTAs each, TMA path), bytes_per_pair = "
                           "multi_bytes; their traffic stays in that GPU's HBM")
    res["multi_bytes"] = a.multi_bytes
    for n in (2, 4):
        cfg = pkg.Config(ordinals=[0] * n, bytes=a.multi_bytes * (n - 1), flags=0x40 | 0x10, ctas=32,
                         timeout_ms=20000)
        with pkg.Open(cfg) as p:
            ts = p.AllReduceTwoShot(a.reps)
            res[f"twoshot_n{n}"] = {**rows(ts, 2 * (n - 1) / n), "call_ms": ts.ms}
res["gpu"] = gpu()
res["nvlink"] = "not measured (one GPU)"

print(f"{'path':8} {'bytes':>12} {'ns_min':>12} {'ns_median':>12} {'ns_max':>12} {'algbw GB/s':>11}")
for name in ("tma", "ldst16", "ldst32"):
    for s in res[f"n1_{name}"]["rank_0"]["sizes"]:
        print(f"{name:8} {s['bytes']:12d} {s['ns_min']:12.0f} {s['ns_median']:12.0f} {s['ns_max']:12.0f} "
              f"{s['algbw_gbps_median']:11.1f}")
if a.twoshot:
    print(f"\n{'two-shot':12} {'rank':>4} {'bytes':>12} {'ns_median':>12} {'algbw GB/s':>11} {'busbw GB/s':>11}")
    for key in [f"twoshot_n1_{x}" for x in ("tma", "ldst16", "ldst32")] + ["twoshot_n2", "twoshot_n4"]:
        for rk, row in res[key].items():
            if not rk.startswith("rank_"):
                continue
            for s in row["sizes"]:
                print(f"{key[8:]:12} {rk[5:]:>4} {s['bytes']:12d} {s['ns_median']:12.0f} "
                      f"{s['algbw_gbps_median']:11.1f} {s['busbw_gbps_median']:11.1f}")
print(f"gpu: {res['gpu']}")
if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
print(json.dumps(res))
