"""cdprobe_allreduce_nvls on the GPU.  The data path runs on a team of devices that report multicast support
(CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, read by the module fixture), one rank per device: all of them when there are
two or more, else device 0 alone, if the driver accepts a multicast object of one device.  With such a team: every size
of a 1 GiB ladder is clean and equal to cdprobe_allreduce's on the same handle; tiny ladders with a partial last unit
on small, odd and full grids; a word corrupted at rest fails exactly the sizes that cover it; both fault modes at word
0, the last word of a partial unit and the grid's last warp fail exactly the words the restatement names
(allreduce_nvls_ref); repeated calls stay exact and disturb nothing; open, call and close give back the device memory.
Without one, the data-path tests check that N = 1 reports CDPROBE_ERR_UNSUPPORTED with the reason in
cdprobe_last_error, and skip with it.  Wherever they run: a single rank the driver refuses, ranks sharing one device,
in one process or two, and simulated MIG run nothing and report CDPROBE_ERR_UNSUPPORTED, with the call returning OK
and no NVLS area created.

Not exercisable on one GPU: a team of two or more devices (so the in-switch sum over several members), the export and
import of the multicast handle between processes, fabric handles, and a down probe mapping on its own terms (it needs
two ranks, which on one GPU share the device and are refused for that first)."""
import ctypes as C
import functools
import textwrap

import numpy as np
import pytest

import allreduce_nvls_ref as ref
import allreduce_ref
import word_ref
from conftest import ROOT
from harness import run_children

pytestmark = pytest.mark.gpu

SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
SIMULATE_MIG = 0x200
ERR_ARG, ERR_UNSUPPORTED, ERR_INTEGRITY = -2, -8, -10
PATH_NVLS = 5
U64_MAX = word_ref.U64_MAX
GIB = 1 << 30
EDGE_BPP = 57 * 8192 + 384  # a partial last unit in a partial last granule: ladder 4096 ... 262144, 467328
PER_ROW = ("sum", "xr", "bad_words", "first_bad")
CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED = 132


@pytest.fixture(scope="module")
def team(pkg):
    """The visible devices whose CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED is 1, read through the driver API (at most
    8), and how many devices there are."""
    cu = C.CDLL("libcuda.so.1")
    count = C.c_int()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGetCount(C.byref(count)) == 0
    on_devices = []
    for i in range(count.value):
        dev, on = C.c_int(), C.c_int()
        assert cu.cuDeviceGet(C.byref(dev), i) == 0
        assert cu.cuDeviceGetAttribute(C.byref(on), CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev) == 0
        if on.value == 1:
            on_devices.append(i)
    return on_devices[:8], count.value


def single_rank_call(pkg, nbytes=1 << 20, flags=0):
    """One cdprobe_allreduce_nvls call of a fresh one-rank handle on device 0: (the result, cdprobe_last_error)."""
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes, flags=flags, ctas=8, timeout_ms=20000)) as p:
        ar = p.AllReduceNVLS(reps=1)
        return ar, p._lib.cdprobe_last_error().decode()


@pytest.fixture(scope="module")
def single_rank(pkg):
    return single_rank_call(pkg)


@pytest.fixture
def data_path(team, single_rank):
    """The ordinals of the data-path tests' team: every device with multicast when there are two or more; device 0
    alone when it has multicast and the driver accepts a one-device object.  Otherwise N = 1 reports
    CDPROBE_ERR_UNSUPPORTED, and the test skips with the reason."""
    devs, count = team
    if len(devs) >= 2:
        return devs
    ar, err = single_rank
    if devs == [0] and ar.measured[0]:
        return devs
    assert not ar.measured[0] and ar.status[0] == ERR_UNSUPPORTED and ar.call_seq == 1
    if 0 not in devs:
        assert err == ""  # refused by the capability check: the driver was not asked
        pytest.skip(f"{count} device(s), none reporting CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED = 1: "
                    "CDPROBE_ERR_UNSUPPORTED")
    assert err.startswith("cuMulticastCreate: "), err  # the driver's own refusal, with its CUresult
    pytest.skip(f"one device with multicast, and the driver refuses a multicast object of one device ({err}): "
                "CDPROBE_ERR_UNSUPPORTED")


def open_team(pkg, devs, bpp, ctas=8, timeout_ms=20000):
    """One rank per device, bytes_per_pair bpp (sliced mode: bytes / peers)."""
    n = len(devs)
    p = pkg.Open(pkg.Config(ordinals=devs, bytes=bpp * max(n - 1, 1), ctas=ctas, timeout_ms=timeout_ms))
    assert p.Info().bytes_per_pair == bpp
    return p


def open_same(pkg, n, nbytes=1 << 20, flags=0):
    return pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME | flags, ctas=8, timeout_ms=20000))


@functools.lru_cache(maxsize=None)
def src(rank, n_words):
    w = word_ref.src_words(SEED, rank, 0, n_words)
    w.setflags(write=False)
    return w


def check(ar, n, bpp, reps, corrupt=None, fault=None):
    """Every row at every size: corrupt {(rank, word): mask} is xored into the sources at rest; fault (mode, k, word)
    acts in timed rep 1 only.  bad_words count every rep, warm-up included; (S, X) is the last timed rep's."""
    sizes = allreduce_ref.ladder(bpp)
    assert ar.sizes == sizes and ar.reps == reps and ar.n == n and ar.path == PATH_NVLS
    W = bpp // 8
    srcs = [src(j, W).copy() for j in range(n)]
    for (j, w), m in (corrupt or {}).items():
        srcs[j][w] ^= np.uint64(m)
    clean = sum((src(j, W) for j in range(1, n)), src(0, W).copy())
    at_rest = sum(srcs[1:], srcs[0].copy())
    for r in range(n):
        bits = 0
        for k, s in enumerate(sizes):
            rep_words = at_rest[:s // 8]
            bad = np.flatnonzero(rep_words != clean[:s // 8])
            n_bad, first, last = (reps + 1) * len(bad), [int(bad[0])] if len(bad) else [], rep_words
            if fault is not None and fault[1] == k:
                hit = ref.rep([x[:s // 8] for x in srcs], s, (fault[0], fault[2]))[r]
                hbad = np.flatnonzero(hit != clean[:s // 8])
                n_bad += len(hbad) - len(bad)
                first += [int(hbad[0])] if len(hbad) else []
                if len(hbad):
                    bits |= 1 << k
                if reps == 1:
                    last = hit
            if len(bad):
                bits |= 1 << k
            ctx = (r, s, fault, corrupt)
            assert (ar.sum[r][k], ar.xr[r][k]) == allreduce_ref.checksum(last), ctx
            assert ar.bad_words[r][k] == n_bad, (ctx, ar.bad_words[r][k], n_bad)
            assert ar.first_bad[r][k] == (8 * min(first) if first else U64_MAX), ctx
            assert 0 < ar.ns_min[r][k] <= ar.ns_median[r][k] <= ar.ns_max[r][k], ctx
        assert ar.measured[r] and ar.bad_sizes[r] == bits, (r, ar.bad_sizes[r], bits)
        assert ar.status[r] == (ERR_INTEGRITY if bits else 0), r
        assert (ar.t0_ns[r], ar.peak_gbps[r], ar.half_bytes[r]) == allreduce_ref.summary(sizes, ar.ns_median[r])
    return ar


# ---- with a team of devices that have multicast ---------------------------------------------------------------------
def test_every_size_of_a_1_gib_ladder_clean_and_equal_to_the_one_shot(pkg, data_path):
    n = len(data_path)
    with open_team(pkg, data_path, GIB, ctas=0, timeout_ms=60000) as p:
        p.SetOption(pkg.abi.OPT_PATH, 1)  # ignored: the NVLS all-reduce has one data path
        ar = p.AllReduceNVLS(reps=2)
        assert ar.sizes == allreduce_ref.ladder(GIB) and ar.path == PATH_NVLS and ar.call_seq == 1
        one = p.AllReduce(reps=2)
        for r in range(n):
            assert ar.measured[r] and ar.status[r] == 0 and ar.bad_sizes[r] == 0, r
            assert ar.bad_words[r] == [0] * len(ar.sizes) and ar.first_bad[r] == [U64_MAX] * len(ar.sizes)
            for f in PER_ROW:
                assert getattr(ar, f)[r] == getattr(one, f)[r], (r, f)


@pytest.mark.parametrize("bpp", [128, 4224, 16512, 24704, EDGE_BPP])
def test_tiny_ladders_with_a_partial_last_unit_on_every_grid(pkg, data_path, bpp):
    n = len(data_path)
    with open_team(pkg, data_path, bpp, ctas=0) as p:
        full = p.Info().ctas[0]
        for ctas in (1, 2, 3, 7, 40, full):
            p.SetOption(pkg.abi.OPT_CTAS, ctas)
            check(p.AllReduceNVLS(reps=1), n, bpp, 1)
            check(p.AllReduceNVLS(reps=3), n, bpp, 3)


def test_a_corrupt_word_fails_exactly_the_sizes_that_cover_it(pkg, data_path):
    n, bpp = len(data_path), EDGE_BPP
    W = bpp // 8
    with open_team(pkg, data_path, bpp) as p:
        for j, w in ((0, 5), (n - 1, 40000), (n // 2, W - 1)):
            p.Corrupt(j, 8 * w, 1 << 17)
            check(p.AllReduceNVLS(reps=2), n, bpp, 2, corrupt={(j, w): 1 << 17})
            p.Corrupt(j, 8 * w, 1 << 17)  # restore
        check(p.AllReduceNVLS(reps=1), n, bpp, 1)


def fault_places(bpp, n, ctas):
    """(k, word): word 0, the last word of the partial last unit, and a word of the unit the last warp of the grid of
    the rank that owns unit 8 ctas - 1 takes first, at the largest size."""
    sizes = allreduce_ref.ladder(bpp)
    k = len(sizes) - 1
    W, U = sizes[k] // 8, ref.units(sizes[k])
    out = [(k, 0), (k, W - 1), (max(k - 2, 0), 0)]
    o = ref.owner(U, n, 0)
    last_warp = U * o // n + 8 * ctas - 1  # rank o's chunk starts at unit floor(o U / n)
    if last_warp < U * (o + 1) // n:
        out.append((k, last_warp * ref.UNIT_WORDS + 7))
    return out


@pytest.mark.parametrize("bpp, ctas", [(EDGE_BPP, 2), ((4 << 20) + 384, 8)])
def test_each_fault_fails_exactly_the_words_the_restatement_names(pkg, data_path, bpp, ctas):
    """Mode 0 stores one word xored with 1, mode 1 skips one unit's store, which then reads as the 0s the previous
    check left, in every row.  With reps == 1 the word check and the last (S, X) see it; with 3 reps the summed bad
    words do.  The output is cleared after every rep, so only size[k] fails, and the next call is clean."""
    a = pkg.abi
    n = len(data_path)
    W = bpp // 8
    with open_team(pkg, data_path, bpp, ctas=ctas) as p:
        sizes = allreduce_ref.ladder(bpp)
        places = fault_places(bpp, n, ctas)
        assert len(places) == 4
        for mode in (0, 1):
            for k, word in places:
                p.SetOption(a.OPT_ALLREDUCE_NVLS_FAULT, a.allreduce_nvls_fault(k, word, mode))
                ar = check(p.AllReduceNVLS(reps=1), n, bpp, 1, fault=(mode, k, word))
                rows = ref.failing([src(j, W)[:sizes[k] // 8] for j in range(n)], sizes[k], (mode, word))
                assert sorted(rows) == list(range(n))
                for r in range(n):
                    assert ar.bad_sizes[r] == 1 << k and ar.bad_words[r][k] == len(rows[r])
                    assert ar.first_bad[r][k] == 8 * rows[r][0]
                check(p.AllReduceNVLS(reps=3), n, bpp, 3, fault=(mode, k, word))
        p.SetOption(a.OPT_ALLREDUCE_NVLS_FAULT, 0)
        check(p.AllReduceNVLS(reps=2), n, bpp, 2)


NO_MODE = "the armed NVLS all-reduce fault has a mode above 1"
NO_FIELD = "the armed NVLS all-reduce fault sets bits 32 to 47, which name nothing"
NO_SIZE = "the armed NVLS all-reduce fault names no size of this call"
NO_WORD = "the armed NVLS all-reduce fault names no output word of its size"


def test_an_armed_fault_that_names_nothing_is_refused_with_its_text(pkg):
    """The fault is checked before the domain is: a single rank, which runs nothing, refuses it all the same."""
    a = pkg.abi
    with pkg.Open(pkg.Config(ordinals=[0], bytes=1 << 20, ctas=8, timeout_ms=20000)) as p:
        sizes = allreduce_ref.ladder(p.Info().bytes_per_pair)
        for v, message in [((2 << 48) | a.allreduce_nvls_fault(0, 0), NO_MODE),
                           ((1 << 63) | a.allreduce_nvls_fault(0, 0), NO_MODE),
                           ((1 << 32) | a.allreduce_nvls_fault(0, 0), NO_FIELD),
                           (5, NO_SIZE),
                           (a.allreduce_nvls_fault(len(sizes), 0), NO_SIZE),
                           (a.allreduce_nvls_fault(0, sizes[0] // 8), NO_WORD)]:
            p.SetOption(a.OPT_ALLREDUCE_NVLS_FAULT, v)
            rc, t = p.allreduce_nvls_raw(2)
            assert rc == ERR_ARG and t.call_seq == 0 and sum(t.measured) == 0, hex(v)
            assert p._lib.cdprobe_last_error().decode() == message, hex(v)
        p.SetOption(a.OPT_ALLREDUCE_NVLS_FAULT, a.allreduce_nvls_fault(len(sizes) - 1, 0, 1))
        rc, t = p.allreduce_nvls_raw(2)  # a fault that names a word is accepted
        assert rc == 0 and t.call_seq == 1 and t.status[0] in (ERR_UNSUPPORTED, ERR_INTEGRITY)
        p.SetOption(a.OPT_ALLREDUCE_NVLS_FAULT, 0)
        rc, t = p.allreduce_nvls_raw(a.ALLREDUCE_MAX_REPS + 1)
        assert rc == ERR_ARG and (t.abi, t.n, t.reps, t.call_seq, t.row_mask, t.path) == (2, 1, 65, 0, 0, PATH_NVLS)


def test_repeated_calls_stay_exact_and_disturb_nothing(pkg, oracle, data_path):
    n = len(data_path)
    with open_team(pkg, data_path, 1 << 20, ctas=16) as p:
        bpp = p.Info().bytes_per_pair
        one = p.AllReduce(reps=2)
        ts = p.AllReduceTwoShot(reps=2)
        ring = p.AllReduceRing(reps=2)
        r1 = p.Run()
        for c in range(1, 6):
            assert check(p.AllReduceNVLS(reps=1 + c % 3), n, bpp, 1 + c % 3).call_seq == c
        for fn, before in ((p.AllReduce, one), (p.AllReduceTwoShot, ts), (p.AllReduceRing, ring)):
            after = fn(reps=2)
            assert after.call_seq == 2 and [getattr(after, f) for f in PER_ROW + ("status",)] == \
                [getattr(before, f) for f in PER_ROW + ("status",)]
        r2 = p.Run()
        assert r2.run_seq == r1.run_seq + 1 and r2.reach == r1.reach and not r2.aborted
        assert (r2.sum_read, r2.xor_read) == (r1.sum_read, r1.xor_read)
        assert check(p.AllReduceNVLS(reps=2), n, bpp, 2).call_seq == 6


def free_bytes(ordinal=0):
    import torch
    torch.cuda.synchronize(ordinal)
    return torch.cuda.mem_get_info(ordinal)[0]


def test_open_call_and_close_give_back_the_device_memory(pkg, data_path):
    n = len(data_path)

    def cycle():
        with open_team(pkg, data_path, 64 << 20) as p:
            check(p.AllReduceNVLS(reps=1), n, 64 << 20, 1)
    cycle()  # the first cycle loads the kernels
    start = free_bytes(data_path[0])
    for _ in range(3):
        cycle()
    assert free_bytes(data_path[0]) >= start - (2 << 20)  # an NVLS area left behind would hold 128 MiB


# ---- wherever it runs ---------------------------------------------------------------------------------------------
def assert_runs_nothing(ar, n, status=ERR_UNSUPPORTED):
    assert ar.n == n and ar.path == PATH_NVLS and ar.call_seq >= 1 and ar.ms < 5000
    for r in range(n):
        assert not ar.measured[r] and ar.ns_median[r] is None and ar.status[r] == status, r


@pytest.mark.parametrize("n", [2, 3, 8])
def test_ranks_sharing_a_device_run_nothing_and_create_nothing(pkg, n):
    """A multicast team holds each device once: ranks on one device could never all join the object."""
    with open_same(pkg, n, nbytes=64 << 20) as p:
        start = free_bytes()
        for c in (1, 2):
            assert_runs_nothing(p.AllReduceNVLS(reps=2), n)
        assert free_bytes() >= start - (2 << 20)  # no NVLS area: it would take 128 MiB per rank
        check_one = p.AllReduce(reps=1)  # the handle is unharmed
        assert all(check_one.status[r] == 0 for r in range(n))


def test_a_single_rank_the_driver_refuses_runs_nothing_and_keeps_nothing(pkg, team, single_rank):
    """Where device 0 has multicast but the driver refuses a multicast object of one device, every call asks again,
    names the driver's CUresult, reports CDPROBE_ERR_UNSUPPORTED and keeps no memory."""
    if 0 not in team[0] or single_rank[0].measured[0]:
        pytest.skip("device 0 has no multicast, or the driver accepts a one-device object (the data-path tests run)")
    with pkg.Open(pkg.Config(ordinals=[0], bytes=64 << 20, ctas=8, timeout_ms=20000)) as p:
        start = free_bytes()
        for c in (1, 2):
            ar = p.AllReduceNVLS(reps=2)
            assert_runs_nothing(ar, 1)
            assert ar.call_seq == c and ar.row_mask == 1 and ar.sizes == allreduce_ref.ladder(64 << 20)
            assert p._lib.cdprobe_last_error().decode().startswith("cuMulticastCreate: ")
        assert free_bytes() >= start - (2 << 20)  # an NVLS area would take 128 MiB
        assert p.AllReduce(reps=1).status[0] == 0


def test_simulated_mig_runs_nothing_before_the_driver_is_asked(pkg):
    """A single simulated MIG instance is refused by the capability check itself: the driver is never asked, so no
    CUresult is named (a one-rank domain that reached cuMulticastCreate would name it)."""
    ar, err = single_rank_call(pkg, flags=SIMULATE_MIG)
    assert_runs_nothing(ar, 1)
    assert err == ""


def test_shared_device_rules_decide_mig_and_down_mapping_domains_of_several_ranks(pkg):
    """With several ranks on one GPU, simulated MIG and a down mapping also run nothing, but the shared-device rule
    decides these domains first: this checks only that nothing runs, not the MIG or mapping rule on its own terms."""
    with open_same(pkg, 2, flags=SIMULATE_MIG) as p:
        assert_runs_nothing(p.AllReduceNVLS(reps=2), 2)
    with open_same(pkg, 3) as p:
        p.UnmapPeer(2, 1)
        assert_runs_nothing(p.AllReduceNVLS(reps=2), 3)
        p.RemapPeer(2, 1)
        assert_runs_nothing(p.AllReduceNVLS(reps=2), 3)


CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    session, rank, world, n_local = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
    cfg = m.Config(ordinals=[0] * n_local, bytes=1 << 20, world_size=world, rank=rank, session=session,
                   flags=0x40 | (0x10 if n_local > 1 else 0), ctas=8, timeout_ms=30000)
    with m.Open(cfg) as p:
        calls = []
        for _ in range(2):
            rc, t = p.allreduce_nvls_raw(2)
            calls.append({"rc": rc, "call_seq": t.call_seq, "row_mask": t.row_mask, "path": t.path,
                          "measured": list(t.measured)[:world * n_local], "status": list(t.status)[:world * n_local]})
        one = p.AllReduce(reps=1)
        print("RESULT " + json.dumps({"calls": calls, "one_status": one.status}))
    """
) % ROOT


@pytest.mark.parametrize("n_local", [1, 2], ids=["2x1", "2x2"])
def test_two_processes_sharing_a_device_agree_to_run_nothing(pkg, n_local):
    """Both processes drive GPU 0: their ranks' UUIDs are equal across processes, so every process refuses alike."""
    world = 2
    n = world * n_local
    outs = run_children(CHILD, world, n_local)
    for rank, o in enumerate(outs):
        mine = set(range(rank * n_local, (rank + 1) * n_local))
        assert [c["call_seq"] for c in o["calls"]] == [1, 2]
        for c in o["calls"]:
            assert c["rc"] == 0 and c["path"] == PATH_NVLS and c["row_mask"] == sum(1 << r for r in mine)
            assert c["measured"] == [0] * n
            assert [c["status"][r] for r in sorted(mine)] == [ERR_UNSUPPORTED] * n_local
        assert all(o["one_status"][r] == 0 for r in mine)
