"""cdprobe_ce_alltoall on the GPU: every block of every domain shape lands every word of every size, pulled and pushed,
with the (S, X) of the pattern, and every block is word-checked by its owner; each rank's rep contains its copies; a
process that would share hardware queues is refused and keeps its handle; an armed fault fails exactly its cell and
size, or only delays it, and the next call is clean; a mapping that is down runs nothing; the neighbouring measurements
stay clean; two processes give what one gives; and nothing leaks.  Several ranks share one device; domains whose
streams exceed the default 8 hardware queues run in child processes with CUDA_DEVICE_MAX_CONNECTIONS=32, and three
ranks run at exactly the queues they need, and are refused one queue below, in children with the limit set so."""
import json
import os
import subprocess
import sys
import textwrap

import pytest

import ce_alltoall_ref as ref
from conftest import ROOT
from harness import run_children

pytestmark = pytest.mark.gpu

SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE
LOCAL_DIAG = 0x4
SIMULATE_MIG = 0x200
MODE_SLICED, MODE_FULL = 1, 2
OPS = (ref.OP_READ, ref.OP_WRITE)
ERR_UNSUPPORTED, ERR_STATE, ERR_INTEGRITY = -8, -9, -10
U64_MAX = (1 << 64) - 1
GIB = 1 << 30
EVENT_NS = 1000  # CUDA events resolve about 0.5 us


def open_same(pkg, n, flags=0, nbytes=1 << 20, mode=MODE_SLICED):
    return pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, mode=mode, flags=SAME | flags, ctas=8,
                               timeout_ms=20000))


def as_dict(ca):
    return {k: getattr(ca, k) for k in ("n", "row_mask", "reps", "op", "call_seq", "sizes", "measured", "status",
                                         "blocks", "ns_median", "ns_max", "cell_measured", "cell_status", "bad_sizes",
                                         "copy_ns_median", "bad_words", "first_bad", "sum", "xr", "ms")}


def check_call(c, oracle, bpp, mode, diag, skip=()):
    """Every block a local rank owns is checked and clean and has the pattern's (S, X), except the cells in `skip`;
    every local rank ran, issued its cells, and its median rep contains the median copy of each of them."""
    n, k, mine = c["n"], len(c["sizes"]), c["row_mask"]
    cells = ref.cells(n, diag)
    for g, j in cells:
        if mine >> ref.owner(c["op"], g, j) & 1 and (g, j) not in skip:
            assert c["cell_measured"][g][j] and c["cell_status"][g][j] == 0 and c["bad_sizes"][g][j] == 0, \
                (g, j, c["cell_status"][g][j], c["bad_sizes"][g][j])
            assert c["bad_words"][g][j] == [0] * k and c["first_bad"][g][j] == [U64_MAX] * k, (g, j)
            assert [tuple(x) for x in zip(c["sum"][g][j], c["xr"][g][j])] == \
                ref.expected(oracle, SEED, n, bpp, mode, c["op"], g, j, c["sizes"]), (g, j)
        elif not mine >> ref.owner(c["op"], g, j) & 1:
            assert not c["cell_measured"][g][j] and c["sum"][g][j] is None
    for r in range(n):
        if not mine >> r & 1:
            assert not c["measured"][r] and c["ns_median"][r] is None
            continue
        issued = [j for g, j in cells if g == r]
        assert c["measured"][r] and c["status"][r] == 0 and c["blocks"][r] == len(issued)
        assert all(t > 0 for t in c["ns_median"][r])
        for j in issued:
            for s in range(k):
                assert c["ns_median"][r][s] >= c["copy_ns_median"][r][j][s] - EVENT_NS, (r, j, s)
    assert max(sum(c["ns_median"][r]) for r in range(n) if mine >> r & 1) / 1e6 <= c["ms"]


@pytest.mark.parametrize("op", OPS, ids=["pull", "push"])
@pytest.mark.parametrize("nbytes", [4 << 20, GIB], ids=["4MiB", "1GiB"])
def test_single_rank_every_size_clean(pkg, oracle, nbytes, op):
    reps = 8 if nbytes < GIB else 2
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes, timeout_ms=20000)) as p:
        ca = p.CeAllToAll(op, reps)
        assert (ca.n, ca.row_mask, ca.reps, ca.op, ca.call_seq) == (1, 1, reps, op, 1)
        assert ca.area_bytes == (nbytes + (2 << 20) - 1) // (2 << 20) * (2 << 20)
        assert ca.sizes == ref.ladder(nbytes)
        check_call(as_dict(ca), oracle, nbytes, MODE_SLICED, True)
        ca2 = p.CeAllToAll(op, reps=1)
        assert ca2.call_seq == 2
        check_call(as_dict(ca2), oracle, nbytes, MODE_SLICED, True)


CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path[:0] = [%r, %r]
    import cdprobe_pkg
    import test_ce_alltoall_gpu as t
    m = cdprobe_pkg.load()
    session, rank, world, n_local = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
    out = []
    for mode in (1, 2):
        for diag in (0, 4):
            cfg = m.Config(ordinals=[0] * n_local, bytes=1 << 20, mode=mode, world_size=world, rank=rank,
                           session=f"{session}-{mode}-{diag}", flags=0x50 | diag, ctas=8, timeout_ms=30000)
            with m.Open(cfg) as p:
                for op in (m.abi.OP_READ, m.abi.OP_WRITE):
                    out.append({"mode": mode, "diag": diag, **t.as_dict(p.CeAllToAll(op, reps=2))})
    print("RESULT " + json.dumps(out))
    """
) % (ROOT, os.path.join(ROOT, "tests"))


@pytest.mark.parametrize("world,n_local", [(1, 2), (1, 3), (1, 4), (4, 2)], ids=["2", "3", "4", "8=4x2"])
def test_every_block_of_every_domain_clean(pkg, oracle, monkeypatch, world, n_local):
    """Sliced and full, with and without LOCAL_DIAG, pulled and pushed: every block is checked by its owner's process
    and clean, and every rank's rep contains its copies."""
    monkeypatch.setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    n = world * n_local
    outs = run_children(CHILD, world, n_local)
    for rank, calls in enumerate(outs):
        assert len(calls) == 8
        for c in calls:
            assert c["row_mask"] == ((1 << n_local) - 1) << (rank * n_local) and c["n"] == n
            bpp = pkg.plan(n, 1 << 20, c["mode"], c["diag"]).bytes_per_pair
            check_call(c, oracle, bpp, c["mode"], bool(c["diag"]))
    # every block of the domain was checked by exactly one process
    for c0 in range(8):
        for g, j in ref.cells(n, bool(outs[0][c0]["diag"])):
            assert sum(o[c0]["cell_measured"][g][j] for o in outs) == 1, (c0, g, j)


def test_too_many_streams_for_the_hardware_queues_is_refused(pkg, oracle):
    """Eight ranks on one device need 8 x 8 streams: more than CUDA_DEVICE_MAX_CONNECTIONS gives, so the call is
    refused with the need and the limit named, and the handle stays usable."""
    limit = max(1, min(32, int(os.environ.get("CUDA_DEVICE_MAX_CONNECTIONS") or 8)))
    n = 8
    with open_same(pkg, n) as p:
        rc, t = p.ce_alltoall_raw(ref.OP_WRITE, 2)
        assert rc == ERR_UNSUPPORTED and t.call_seq == 0 and sum(t.measured) == 0 and t.n == n
        assert ref.queue_message(64, 0, limit) in pkg.abi.load_library().cdprobe_last_error().decode()
        with pytest.raises(pkg.ErrUnsupported):
            p.CeAllToAll(ref.OP_READ, 2)
        aa = p.AllToAll(reps=1)
        assert all(aa.cell_status[s][d] == 0 for s in range(n) for d in range(n) if s != d)
        r = p.Run()
        assert r.reach == [[1] * n for _ in range(n)] and not r.aborted


@pytest.mark.parametrize("op", OPS, ids=["pull", "push"])
@pytest.mark.parametrize("mode", [0, 1, 2], ids=["flip", "drop", "hold"])
def test_an_armed_fault_acts_on_exactly_its_cell_and_size(pkg, oracle, mode, op):
    n, nbytes, k, g, j = 2, 1 << 20, 2, 0, 1
    a = pkg.abi
    with open_same(pkg, n, nbytes=nbytes) as p:
        bpp = pkg.plan(n, nbytes, MODE_SLICED).bytes_per_pair
        sizes = ref.ladder(bpp)
        arg = 5 if mode < 2 else 3000
        p.SetOption(a.OPT_CE_ALLTOALL_FAULT, a.ce_alltoall_fault(g, j, k, arg, mode))
        c = as_dict(p.CeAllToAll(op, reps=2))
        if mode == 2:
            check_call(c, oracle, bpp, MODE_SLICED, False)
            recv = ref.owner(op, g, j)
            assert c["ns_max"][recv][k] >= arg * 1000 - 20_000, c["ns_max"][recv][k]  # less the opening barrier
        else:
            check_call(c, oracle, bpp, MODE_SLICED, False, skip={(g, j)})
            assert c["cell_measured"][g][j] and c["cell_status"][g][j] == ERR_INTEGRITY
            assert c["bad_sizes"][g][j] == 1 << k
            words, first = ref.fault_words(mode, sizes[k], arg)
            assert c["bad_words"][g][j] == [words if s == k else 0 for s in range(len(sizes))]
            assert c["first_bad"][g][j] == [first if s == k else U64_MAX for s in range(len(sizes))]
            # the last timed rep is clean again: the owner cleared the block, and the next rep landed it whole
            assert [tuple(x) for x in zip(c["sum"][g][j], c["xr"][g][j])] == \
                ref.expected(oracle, SEED, n, bpp, MODE_SLICED, op, g, j, sizes)
        p.SetOption(a.OPT_CE_ALLTOALL_FAULT, 0)
        check_call(as_dict(p.CeAllToAll(op, reps=2)), oracle, bpp, MODE_SLICED, False)


def test_a_fault_that_names_nothing_of_the_call_is_refused(pkg, oracle):
    n, nbytes = 2, 1 << 20
    a = pkg.abi
    with open_same(pkg, n, nbytes=nbytes) as p:
        sizes = ref.ladder(pkg.plan(n, nbytes, MODE_SLICED).bytes_per_pair)
        for bad in (a.ce_alltoall_fault(n, 0, 0, 0), a.ce_alltoall_fault(1, 1, 0, 0),
                    a.ce_alltoall_fault(0, 1, len(sizes), 0), a.ce_alltoall_fault(0, 1, 0, sizes[0] // 8),
                    a.ce_alltoall_fault(0, 1, 0, 10_000_000, mode=2), (3 << 48) | (1 << 40) | (2 << 32) | (1 << 24)):
            p.SetOption(a.OPT_CE_ALLTOALL_FAULT, bad)
            rc, t = p.ce_alltoall_raw(ref.OP_WRITE, 2)
            assert rc == -2 and t.call_seq == 0 and sum(t.measured) == 0
            assert (t.abi, t.n, t.reps, t.op) == (2, n, 2, ref.OP_WRITE)
        # a delay below timeout_ms / 2 and a word past the smallest size but inside its own are accepted
        p.SetOption(a.OPT_CE_ALLTOALL_FAULT, a.ce_alltoall_fault(0, 1, 1, sizes[0] // 8, mode=2))
        assert p.CeAllToAll(ref.OP_READ, 1).call_seq == 1
        p.SetOption(a.OPT_CE_ALLTOALL_FAULT, 0)
        check_call(as_dict(p.CeAllToAll(ref.OP_READ, 1)), oracle, nbytes, MODE_SLICED, False)


@pytest.mark.parametrize("op", OPS, ids=["pull", "push"])
def test_a_mapping_that_is_down_runs_nothing(pkg, oracle, op):
    n, nbytes = 2, 1 << 20
    with open_same(pkg, n, nbytes=nbytes) as p:
        check_call(as_dict(p.CeAllToAll(op, reps=1)), oracle, nbytes, MODE_SLICED, False)
        p.UnmapPeer(1, 0)
        ca = p.CeAllToAll(op, reps=1)
        assert ca.call_seq == 2 and ca.measured == [False, False] and ca.status == [ERR_STATE, ERR_STATE]
        assert not any(ca.cell_measured[s][d] for s in range(n) for d in range(n))
        assert ca.cell_status[0][1] == ERR_STATE and ca.cell_status[1][0] == ERR_STATE
        p.RemapPeer(1, 0)
        check_call(as_dict(p.CeAllToAll(op, reps=1)), oracle, nbytes, MODE_SLICED, False)


def test_simulated_mig_runs_nothing(pkg):
    with open_same(pkg, 2, flags=SIMULATE_MIG) as p:
        for call, op in enumerate(OPS, 1):
            ca = p.CeAllToAll(op, reps=1)
            assert ca.call_seq == call and ca.measured == [False, False]
            assert ca.status == [ERR_UNSUPPORTED, ERR_UNSUPPORTED] and ca.ns_median == [None, None]


def test_the_neighbouring_measurements_stay_clean(pkg, oracle):
    n, nbytes = 2, 1 << 20
    with open_same(pkg, n, nbytes=nbytes) as p:
        r1 = p.Run()
        assert r1.reach == [[1] * n for _ in range(n)] and not r1.aborted
        diags = {(op, i, j): p.Diagnose(op, i, j) for i, j in ((0, 1), (1, 0)) for op in ("read", "write")}
        aa = p.AllToAll(reps=2)
        mc = p.Memcpy(ref.OP_WRITE, reps=2)
        for op in OPS:
            check_call(as_dict(p.CeAllToAll(op, reps=2)), oracle, nbytes, MODE_SLICED, False)
        for key, d in diags.items():
            d2 = p.Diagnose(*key)
            assert d2.bad_words == 0 and (d2.run_seq, d2.region_offset) == (d.run_seq, d.region_offset), key
        aa2 = p.AllToAll(reps=2)
        assert aa2.area_bytes == aa.area_bytes
        assert all(aa2.cell_status[s][d] == 0 and aa2.bad_sizes[s][d] == 0 for s in range(n) for d in range(n) if s != d)
        mc2 = p.Memcpy(ref.OP_WRITE, reps=2)
        assert all(mc2.status[s][d] == 0 and mc2.sum[s][d] == mc.sum[s][d] for s in range(n) for d in range(n) if s != d)
        r2 = p.Run()
        assert r2.run_seq == r1.run_seq + 1 and r2.reach == r1.reach and not r2.aborted
        assert (r2.sum_read, r2.xor_read) == (r1.sum_read, r1.xor_read)
        words = r2.bytes_per_pair // 8
        for i, j in ((0, 1), (1, 0)):
            assert (r2.sum_write[i][j], r2.xor_write[i][j]) == oracle.write_checksum(SEED, i, j, r2.run_seq, words)


TWO = textwrap.dedent(
    """
    import json, sys
    sys.path[:0] = [%r, %r]
    import cdprobe_pkg
    import test_ce_alltoall_gpu as t
    m = cdprobe_pkg.load()
    session, rank, world = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    cfg = m.Config(ordinals=[0], bytes=1 << 20, world_size=world, rank=rank, session=session, flags=0x40,
                   ctas=8, timeout_ms=30000)
    with m.Open(cfg) as p:
        out = [t.as_dict(p.CeAllToAll(op, reps=2)) for op in (m.abi.OP_READ, m.abi.OP_WRITE)]
    print("RESULT " + json.dumps(out))
    """
) % (ROOT, os.path.join(ROOT, "tests"))


def test_two_processes_give_the_cells_of_one(pkg, oracle):
    n = 2
    outs = run_children(TWO, n)
    with open_same(pkg, n) as p:
        one = [as_dict(p.CeAllToAll(op, reps=2)) for op in OPS]
    for call in range(2):
        for rank, o in enumerate(outs):
            c = o[call]
            assert c["row_mask"] == 1 << rank and c["call_seq"] == call + 1
            check_call(c, oracle, 1 << 20, MODE_SLICED, False)
            for g, j in ref.cells(n, False):
                if ref.owner(c["op"], g, j) == rank:
                    for f in ("cell_status", "bad_sizes", "bad_words", "first_bad", "sum", "xr"):
                        assert c[f][g][j] == one[call][f][g][j], (f, g, j)


def test_no_leak(pkg):
    import torch
    nbytes = 64 << 20
    torch.cuda.init()
    free0 = torch.cuda.mem_get_info(0)[0]
    fds0 = len(os.listdir("/proc/self/fd"))
    for _ in range(3):
        with open_same(pkg, 2, nbytes=nbytes) as p:
            p.CeAllToAll(ref.OP_READ, reps=1)
            free1 = torch.cuda.mem_get_info(0)[0]
            fds1 = len(os.listdir("/proc/self/fd"))
            p.CeAllToAll(ref.OP_WRITE, reps=1)
            p.CeAllToAll(ref.OP_READ, reps=1)
            assert torch.cuda.mem_get_info(0)[0] == free1 and len(os.listdir("/proc/self/fd")) == fds1
        assert torch.cuda.mem_get_info(0)[0] == free0
    assert len(os.listdir("/proc/self/fd")) == fds0


# ---- the queue refusal at its edge ----------------------------------------------------------------------------------
BOUNDARY = textwrap.dedent(
    """
    import json, sys
    sys.path[:0] = [%r, %r]
    sys.modules["torch"] = None
    import cdprobe_pkg
    from oracle import oracle
    import test_ce_alltoall_gpu as t
    t.case_boundary(cdprobe_pkg.load(), oracle, *json.loads(sys.argv[1]))
    print("CHILD OK")
    """
) % (ROOT, os.path.join(ROOT, "tests"))


def case_boundary(pkg, oracle, diag, limit):
    """Three ranks on one device, each with its own stream and a copy stream per cell it issues: 9 queues, 12 with
    LOCAL_DIAG.  At need = limit every stream has a hardware queue of its own and both ops run clean; one queue less
    is refused with the need and the limit named, advances nothing, and memcpy still runs clean on the handle."""
    n, nbytes = 3, 1 << 20
    need, ordinal = ref.queues(n, bool(diag), [0] * n)
    assert (need, ordinal) == (9 if not diag else 12, 0)
    with open_same(pkg, n, flags=diag, nbytes=nbytes) as p:
        bpp = pkg.plan(n, nbytes, MODE_SLICED, diag).bytes_per_pair
        if limit >= need:
            for call, op in enumerate(OPS, 1):
                c = as_dict(p.CeAllToAll(op, reps=2))
                assert (c["call_seq"], c["reps"]) == (call, 2)
                check_call(c, oracle, bpp, MODE_SLICED, bool(diag))
            return
        for op in OPS:
            rc, t = p.ce_alltoall_raw(op, 2)
            assert rc == ERR_UNSUPPORTED and t.call_seq == 0 and sum(t.measured) == 0, rc
            assert ref.queue_message(need, 0, limit) in pkg.abi.load_library().cdprobe_last_error().decode()
        mc = p.Memcpy(ref.OP_WRITE, reps=1)
        assert mc.call_seq == 1
        assert all(mc.status[g][j] == 0 and mc.bad_sizes[g][j] == 0 for g, j in ref.cells(n, bool(diag)))


BOUNDARY_CASES = [(0, 9), (0, 8), (LOCAL_DIAG, 12), (LOCAL_DIAG, 11)]


@pytest.mark.parametrize("diag,limit", BOUNDARY_CASES, ids=["9-of-9", "9-of-8", "diag-12-of-12", "diag-12-of-11"])
def test_three_ranks_run_at_exactly_their_queues_and_are_refused_one_below(pkg, oracle, diag, limit):
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS=str(limit))
    pr = subprocess.run([sys.executable, "-c", BOUNDARY, json.dumps([diag, limit])], env=env, capture_output=True,
                        text=True, timeout=600)
    assert pr.returncode == 0 and "CHILD OK" in pr.stdout, pr.stderr[-8000:]
