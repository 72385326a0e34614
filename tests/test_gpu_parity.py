"""Parity tests proper: the CUDA probe (through the C ABI, ctypes) against the CPU oracle.

Bit-exact bar: reachability bits, (S, X) checksums of every slice read or written, the
published source checksums.  GB/s values are measurements (positive, finite; +-2 % run to
run is checked by bench.py, not here).

Small sizes are compared with the oracle's scalar restatement; BASELINE.json's full sizes
(1 GiB, 64 MiB) through the same checksums (the oracle streams 1 GiB in about a second) plus
size-independent properties: write->verify round trip, corruption is detected, a torn-down
mapping yields a 0 cell and the run still returns, run_seq salts make stale data fail.
"""
import json
import subprocess
import sys
import textwrap
import uuid

import pytest

from conftest import ROOT, gpu_count

pytestmark = pytest.mark.gpu

NGPU = gpu_count()
SEED = 0xCD5EED0000000001
SAME = 0x40 | 0x10  # ALLOW_SAME_DEVICE | NO_COOPERATIVE: several ranks on one device


def expected_read(oracle, n, nbytes, mode, i, j, diag=False):
    return oracle.expected_read(SEED, n, nbytes, mode, i, j, diag)


def check_full_parity(pkg, oracle, res, n, nbytes, mode, ops, diag=False):
    bpp = res.bytes_per_pair
    assert bpp == oracle.plan(n, nbytes, mode, diag).bytes_per_pair
    for i in range(n):
        if not (res.row_mask >> i) & 1:
            continue
        for j in range(n):
            if i == j and not (diag or n == 1):
                assert res.reach_read[i][j] == 1 and res.reach_write[i][j] == 1
                continue
            if ops & pkg.abi.OP_READ:
                assert res.reach_read[i][j] == 1, (i, j)
                assert (res.sum_read[i][j], res.xor_read[i][j]) == expected_read(oracle, n, nbytes, mode, i, j, diag), (i, j)
                assert res.gbps_read[i][j] > 0
            if ops & pkg.abi.OP_WRITE:
                assert res.reach_write[i][j] == 1, (i, j)
                exp = oracle.write_checksum(SEED, i, j, res.run_seq, bpp // 8)
                assert (res.sum_write[i][j], res.xor_write[i][j]) == exp, (i, j)
                assert res.gbps_write[i][j] > 0


# ------------------------------------------------------------------ N = 1 loop-back ----
@pytest.mark.parametrize("path_flag", [0, 0x08], ids=["tma", "ldst"])
@pytest.mark.parametrize("nbytes", [128, 8192, 8192 + 128, 16384 * 3 + 640, 1 << 20, (1 << 23) + 128 * 77])
def test_single_gpu_small_sizes(pkg, oracle, nbytes, path_flag):
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes, mode=pkg.abi.MODE_SLICED, flags=path_flag)) as p:
        info = p.Info()
        assert info.n == 1 and info.n_slices == 1
        exp = oracle.src_checksum(SEED, 0, 0, nbytes // 128 * 128 // 8)
        assert (info.src_sum[0][0], info.src_xor[0][0]) == exp  # device-published == oracle
        for _ in range(3):
            r = p.Run()
            assert r.verdict and not r.aborted and r.launches == 1
            check_full_parity(pkg, oracle, r, 1, nbytes, pkg.abi.MODE_SLICED, 3)


@pytest.mark.parametrize("path_flag", [0, 0x08], ids=["tma", "ldst"])
def test_single_gpu_one_gib(pkg, oracle, path_flag):
    """BASELINE config at one GPU: 1 GiB buffer, read + write + verify, checksums bit-exact."""
    nbytes = 1 << 30
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes, flags=path_flag)) as p:
        r = p.Run()
        check_full_parity(pkg, oracle, r, 1, nbytes, pkg.abi.MODE_SLICED, 3)
        assert r.verdict
        r2 = p.Run()
        # a new run re-salts the write pattern: same read checksums, different write checksums
        assert r2.sum_read[0][0] == r.sum_read[0][0] and r2.sum_write[0][0] != r.sum_write[0][0]
        check_full_parity(pkg, oracle, r2, 1, nbytes, pkg.abi.MODE_SLICED, 3)


@pytest.mark.parametrize("nbytes", [128, 8192 + 128, 16384 * 3 + 640, (1 << 23) + 128 * 77, 1 << 28])
def test_path_ldst256_single_gpu(pkg, oracle, nbytes):
    """Third data path: 32 contiguous bytes per lane (two 128-bit LDG/STG), selected at run time."""
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes)) as p:
        p.SetOption(pkg.abi.OPT_PATH, 2)
        assert p.Info().path == 2
        for _ in range(2):
            r = p.Run()
            assert r.verdict
            check_full_parity(pkg, oracle, r, 1, nbytes, pkg.abi.MODE_SLICED, 3)


@pytest.mark.parametrize("n", [2, 3, 4])
def test_path_ldst256_same_device_ranks(pkg, oracle, n):
    nbytes = (2 << 20) + 128 * 9
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=8, timeout_ms=20000)) as p:
        p.SetOption(pkg.abi.OPT_PATH, 2)
        r = p.Run()
        check_full_parity(pkg, oracle, r, n, nbytes, pkg.abi.MODE_SLICED, 3)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("ops", [1, 2, 3])
def test_single_gpu_modes_and_ops(pkg, oracle, mode, ops):
    nbytes = 4 << 20
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes, mode=mode, ops=ops)) as p:
        r = p.Run()
        check_full_parity(pkg, oracle, r, 1, nbytes, mode, ops)


def test_corruption_is_detected(pkg, oracle):
    nbytes = 1 << 20
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes)) as p:
        assert p.Run().verdict
        p.Corrupt(0, 4096 + 8, 1 << 17)  # flip one bit of one word of the source buffer
        r = p.Run()
        assert r.reach_read[0][0] == 0 and r.reach_write[0][0] == 1 and not r.verdict
        p.Corrupt(0, 4096 + 8, 1 << 17)  # flip it back
        assert p.Run().verdict


def test_small_grid_and_many_runs(pkg, oracle):
    """Storm-lite (config 5): one handle, many runs, a non-default grid; results stay exact."""
    nbytes = 3 << 20
    with pkg.Open(pkg.Config(ordinals=[0], bytes=nbytes, ctas=5)) as p:
        assert p.Info().ctas[0] == 5
        seqs = []
        for _ in range(40):
            r = p.Run()
            seqs.append(r.run_seq)
            assert r.verdict
        assert seqs == list(range(seqs[0], seqs[0] + 40))
        check_full_parity(pkg, oracle, r, 1, nbytes, pkg.abi.MODE_SLICED, 3)


# --------------------------------------------- several ranks on one device (one process) ----


@pytest.mark.parametrize("path_flag", [0, 0x08], ids=["tma", "ldst"])
@pytest.mark.parametrize("n,mode", [(2, 1), (2, 2), (3, 1), (4, 1), (4, 0), (5, 1), (8, 1)])
def test_same_device_ranks(pkg, oracle, n, mode, path_flag):
    """The whole multi-rank machinery (tournament, peer mappings, cross-rank flag barrier,
    write -> publish -> verify -> verdict) with every rank on GPU 0: works on a 1-GPU box."""
    nbytes = 2 << 20
    cfg = pkg.Config(ordinals=[0] * n, bytes=nbytes, mode=mode, flags=SAME | path_flag, ctas=8, timeout_ms=20000)
    with pkg.Open(cfg) as p:
        for _ in range(2):
            r = p.Run()
            assert r.n == n and r.row_mask == (1 << n) - 1 and r.launches == n
            assert not r.aborted
            check_full_parity(pkg, oracle, r, n, nbytes, mode, 3)
            assert r.reach == [[1] * n for _ in range(n)]
            assert r.rounds == (n if n % 2 else n - 1)


@pytest.mark.parametrize("n", [2, 3, 4, 5, 8])
@pytest.mark.parametrize("flags", [0x80, 0x20, 0xA0], ids=["unidirectional", "overlap-verify", "uni+overlap"])
def test_schedule_variants_keep_parity(pkg, oracle, n, flags):
    """Unidirectional half-rounds and the overlapped verify only reorder phases: every checksum
    and reachability bit must be unchanged."""
    nbytes = 2 << 20
    cfg = pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME | flags, ctas=8, timeout_ms=20000)
    with pkg.Open(cfg) as p:
        p.SetOption(pkg.abi.OPT_VERIFY_CTAS, 3)
        for _ in range(2):
            r = p.Run()
            assert not r.aborted and r.row_mask == (1 << n) - 1
            check_full_parity(pkg, oracle, r, n, nbytes, pkg.abi.MODE_SLICED, 3)
            assert r.reach == [[1] * n for _ in range(n)]


def test_runtime_options_round_trip(pkg, oracle):
    n, nbytes = 4, 1 << 20
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=8, timeout_ms=20000)) as p:
        base = p.Run()
        for opt, val in ((pkg.abi.OPT_PATH, 1), (pkg.abi.OPT_UNIDIRECTIONAL, 1), (pkg.abi.OPT_OVERLAP_VERIFY, 1),
                         (pkg.abi.OPT_VERIFY_CTAS, 2), (pkg.abi.OPT_CTAS, 6), (pkg.abi.OPT_EVENT_TIMING, 1),
                         (pkg.abi.OPT_PATH, 0), (pkg.abi.OPT_UNIDIRECTIONAL, 0), (pkg.abi.OPT_OVERLAP_VERIFY, 0)):
            p.SetOption(opt, val)
            r = p.Run()
            assert r.sum_read == base.sum_read and r.xor_read == base.xor_read
            check_full_parity(pkg, oracle, r, n, nbytes, pkg.abi.MODE_SLICED, 3)
        assert max(r.event_ms) > 0
        with pytest.raises(pkg.ProbeError):
            p.SetOption(99, 1)


def test_wakeup_phase_is_automatic_and_does_not_change_results(pkg, oracle):
    """Phase 0 (link wake-up) streams bytes only after an idle gap; results are identical either way."""
    import time

    n, nbytes = 4, 1 << 20
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=8, timeout_ms=20000)) as p:
        first = p.Run()
        assert first.warmed  # the first run of a handle is always cold
        again = p.Run()
        assert not again.warmed  # back to back: no wake-up traffic
        time.sleep(0.05)
        cold = p.Run()
        assert cold.warmed
        for r in (first, again, cold):
            check_full_parity(pkg, oracle, r, n, nbytes, pkg.abi.MODE_SLICED, 3)
        assert p.Trace(0)[0]["job0"] == "warm"
        p.SetOption(pkg.abi.OPT_WARMUP, 0)
        time.sleep(0.05)
        assert not p.Run().warmed
        p.SetOption(pkg.abi.OPT_WARMUP, 2)
        assert p.Run().warmed


def test_simulated_mig_domain_is_identity_and_not_a_failure(pkg, oracle):
    """BASELINE config 4 without MIG hardware: no P2P between MIG instances => identity matrix (what the
    NVML oracle says for an all-MIG node, tests/test_oracle_nvml.py::test_all_mig_is_identity), diagonal
    measured through local HBM, the run returns, and the verdict is NOT a failure (SURVEY H8)."""
    n, nbytes = 4, 1 << 20
    flags = SAME | pkg.abi.FLAG_SIMULATE_MIG | pkg.abi.FLAG_LOCAL_DIAG
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=flags, ctas=8, timeout_ms=20000)) as p:
        assert all(p.Info().mig[i] == 1 for i in range(n))
        r = p.Run()
        ident = [[1 if i == j else 0 for j in range(n)] for i in range(n)]
        assert r.reach == ident and not r.aborted and r.verdict
        for i in range(n):
            assert r.gbps_read[i][i] > 0 and r.gbps_write[i][i] > 0
            assert (r.sum_read[i][i], r.xor_read[i][i]) == expected_read(oracle, n, nbytes, 1, i, i, diag=True)
            for j in range(n):
                if i != j:
                    assert r.status[i][j] == pkg.abi.ERR_UNSUPPORTED


def test_device_watchdog_bounds_a_missing_peer(pkg, oracle):
    """A rank that never reaches the barrier must not hang the probe (the readiness probe has a 10 s budget,
    templates/compute-domain-daemon.tmpl.yaml:83): the device watchdog fires after timeout_ms, the call
    returns CDPROBE_ERR_TIMEOUT with aborted = 1 and nothing reachable, and the handle recovers."""
    import time

    n, nbytes = 3, 1 << 20
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=8, timeout_ms=300)) as p:
        assert p.Run().reach == [[1] * n for _ in range(n)]
        p.SetOption(pkg.abi.OPT_DEBUG_SKIP_RANK, 2)  # local rank 1 is never launched
        t0 = time.time()
        r = p.Run(allow_timeout=True)
        assert time.time() - t0 < 5.0
        assert r.aborted and not r.verdict
        assert all(r.reach_read[i][j] == 0 for i in range(n) for j in range(n) if i != j)
        p.SetOption(pkg.abi.OPT_DEBUG_SKIP_RANK, 0)
        good = p.Run()
        assert not good.aborted and good.reach == [[1] * n for _ in range(n)]
        check_full_parity(pkg, oracle, good, n, nbytes, pkg.abi.MODE_SLICED, 3)


def test_same_device_with_diagonal(pkg, oracle):
    n, nbytes = 4, 1 << 20
    cfg = pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME | pkg.abi.FLAG_LOCAL_DIAG, ctas=8, timeout_ms=20000)
    with pkg.Open(cfg) as p:
        r = p.Run()
        check_full_parity(pkg, oracle, r, n, nbytes, pkg.abi.MODE_SLICED, 3, diag=True)


def test_unmapped_peer_gives_zero_cell_and_run_returns(pkg, oracle):
    """Fault injection (SURVEY App. C T2): drop rank 1's mapping of rank 2 => cells (1,2) and
    (2,1) are unreachable (a pair needs both directions for its barrier and verdict), every
    other cell stays 1 and the run still returns; remap heals it."""
    n, nbytes = 4, 1 << 20
    cfg = pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=8, timeout_ms=20000)
    with pkg.Open(cfg) as p:
        assert p.Run().reach == [[1] * n for _ in range(n)]
        p.UnmapPeer(1, 2)
        r = p.Run()
        exp = [[1] * n for _ in range(n)]
        exp[1][2] = exp[2][1] = 0
        assert r.reach == exp and not r.verdict and not r.aborted
        assert r.status[1][2] != 0
        p.RemapPeer(1, 2)
        r = p.Run()
        assert r.reach == [[1] * n for _ in range(n)]
        check_full_parity(pkg, oracle, r, n, nbytes, pkg.abi.MODE_SLICED, 3)


def test_corrupt_one_slice_hits_exactly_one_reader(pkg, oracle):
    n, nbytes = 4, 1 << 20
    cfg = pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=8, timeout_ms=20000)
    with pkg.Open(cfg) as p:
        bpp = p.Info().bytes_per_pair
        # slice 1 of rank 0's source is what rank 2 reads (its slot among rank 0's peers)
        p.Corrupt(0, bpp + 64, 0xFF)
        r = p.Run()
        exp = [[1] * n for _ in range(n)]
        exp[2][0] = 0
        assert r.reach_read == exp
        assert r.reach_write == [[1] * n for _ in range(n)]


# ------------------------------------------------ one process per rank (bench.py's layout) ----
CHILD = textwrap.dedent(
    """
    import json, sys
    sys.path.insert(0, %r)
    import cdprobe_pkg
    m = cdprobe_pkg.load()
    session, rank, world, ordinal, nbytes, flags = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5]), int(sys.argv[6])
    cfg = m.Config(ordinals=[ordinal], bytes=nbytes, world_size=world, rank=rank, session=session, flags=flags,
                   ctas=int(sys.argv[7]), timeout_ms=30000)
    with m.Open(cfg) as p:
        info = p.Info()
        out = []
        for _ in range(2):
            r = p.Run(gather=True)
            out.append({"n": r.n, "row_mask": r.row_mask, "reach_read": r.reach_read, "reach_write": r.reach_write,
                        "sum_read": r.sum_read, "xor_read": r.xor_read, "sum_write": r.sum_write,
                        "xor_write": r.xor_write, "run_seq": r.run_seq, "bpp": r.bytes_per_pair,
                        "verdict": r.verdict, "aborted": r.aborted, "handle_type": info.handle_type})
    print("RESULT " + json.dumps(out))
    """
) % ROOT


def run_world(world, ordinals, nbytes, flags, ctas):
    session = f"g-{uuid.uuid4().hex[:12]}"
    procs = [subprocess.Popen([sys.executable, "-c", CHILD, session, str(r), str(world), str(ordinals[r]), str(nbytes),
                               str(flags), str(ctas)], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
             for r in range(world)]
    outs = []
    for p in procs:
        so, se = p.communicate(timeout=300)
        assert p.returncode == 0, se[-2000:]
        outs.append(json.loads([l for l in so.splitlines() if l.startswith("RESULT ")][-1][7:]))
    return outs


def check_world(oracle, outs, world, nbytes):
    for per_rank in outs:
        for r in per_rank:
            assert r["n"] == world and r["row_mask"] == (1 << world) - 1 and not r["aborted"]
            assert r["handle_type"] == 1  # POSIX fd handles crossed the process boundary
            for i in range(world):
                for j in range(world):
                    if i == j:
                        continue
                    assert r["reach_read"][i][j] == 1 and r["reach_write"][i][j] == 1
                    assert (r["sum_read"][i][j], r["xor_read"][i][j]) == expected_read(oracle, world, nbytes, 1, i, j)
                    assert (r["sum_write"][i][j], r["xor_write"][i][j]) == oracle.write_checksum(
                        SEED, i, j, r["run_seq"], r["bpp"] // 8)
    # after cdprobe_gather every process holds the same matrices
    assert all(o == outs[0] for o in outs[1:])


def test_two_processes_share_one_gpu(pkg, oracle):
    """world_size = 2, both on GPU 0: cuMem fd export/import over the unix socket, peer mapping of an
    imported handle, the flag barrier across two contexts (time-sliced, hence the long timeout)."""
    nbytes = 1 << 20
    outs = run_world(2, [0, 0], nbytes, 0x40, 8)
    check_world(oracle, outs, 2, nbytes)


# ----------------------------------------------------------------- real multi-GPU boxes ----
@pytest.mark.skipif(NGPU < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("path_flag", [0, 0x08], ids=["tma", "ldst"])
def test_multi_gpu_in_process_parity_with_nvml_oracle(pkg, oracle, path_flag):
    """Config 2/3: every visible GPU in one domain; reach_read & reach_write must equal the NVML
    oracle's matrix bit for bit (matched by UUID), checksums equal the pattern oracle."""
    n = min(NGPU, 8)
    nbytes = 64 << 20
    with pkg.Open(pkg.Config(ordinals=list(range(n)), bytes=nbytes, mode=pkg.abi.MODE_SLICED, flags=path_flag,
                             timeout_ms=20000)) as p:
        info = p.Info()
        r = p.Run()
        check_full_parity(pkg, oracle, r, n, nbytes, pkg.abi.MODE_SLICED, 3)
        o = oracle.nvml_poll()
        by_uuid = {u: k for k, u in enumerate(o.uuids())}
        idx = [by_uuid[info.uuid[i].value.decode()] for i in range(n)]
        om = o.reach_matrix()
        exp = [[om[idx[i]][idx[j]] for j in range(n)] for i in range(n)]
        assert r.reach == exp
        assert r.reach == [[1] * n for _ in range(n)]  # an HGX H100 box is fully connected


@pytest.mark.skipif(NGPU < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("mode,flags", [(2, 0), (0, 0), (1, 0x80), (2, 0x80 | 0x100), (1, 0x04)],
                         ids=["full", "reach-only", "sliced-unidirectional", "full-uni-serial", "sliced-diag"])
def test_multi_gpu_modes_on_real_peers(pkg, oracle, mode, flags):
    """Every mode / schedule variant across all visible GPUs over real NVLink: same bit-exact bar."""
    n = min(NGPU, 8)
    nbytes = 16 << 20
    with pkg.Open(pkg.Config(ordinals=list(range(n)), bytes=nbytes, mode=mode, flags=flags, timeout_ms=20000)) as p:
        for _ in range(2):
            r = p.Run()
            assert not r.aborted
            check_full_parity(pkg, oracle, r, n, nbytes, mode, 3, diag=bool(flags & 0x04))
            assert all(r.reach[i][j] == 1 for i in range(n) for j in range(n))


@pytest.mark.skipif(NGPU < 3, reason="needs >= 3 GPUs")
@pytest.mark.parametrize("ordinals", [[0, 1, 2], [2, 0, 1], [1, 2]], ids=["0-1-2", "2-0-1", "1-2"])
def test_odd_sized_and_permuted_domains_on_real_peers(pkg, oracle, ordinals):
    """An odd-sized domain (one rank sits out every round) and rank != ordinal, over real NVLink."""
    n, nbytes = len(ordinals), 24 << 20
    with pkg.Open(pkg.Config(ordinals=ordinals, bytes=nbytes, timeout_ms=20000)) as p:
        info = p.Info()
        assert [info.ordinal[i] for i in range(n)] == ordinals
        r = p.Run()
        assert not r.aborted and r.rounds == (n if n % 2 else n - 1)
        check_full_parity(pkg, oracle, r, n, nbytes, pkg.abi.MODE_SLICED, 3)
        assert r.reach == [[1] * n for _ in range(n)]


@pytest.mark.skipif(NGPU < 2, reason="needs >= 2 GPUs")
def test_config2_two_gpu_64mib_full(pkg, oracle):
    """BASELINE config 2: 2-GPU P2P read/write reachability matrix, 64 MiB buffers, full mode."""
    nbytes = 64 << 20
    flags = pkg.abi.FLAG_FABRIC_HANDLES  # fabric handles iff IMEX channel 0 exists, else plain VMM
    with pkg.Open(pkg.Config(ordinals=[0, 1], bytes=nbytes, mode=pkg.abi.MODE_FULL, flags=flags)) as p:
        r = p.Run()
        check_full_parity(pkg, oracle, r, 2, nbytes, pkg.abi.MODE_FULL, 3)
        assert r.reach == [[1, 1], [1, 1]] and r.rounds == 1


@pytest.mark.skipif(NGPU < 2, reason="needs >= 2 GPUs")
def test_multi_gpu_one_process_per_gpu(pkg, oracle):
    n = min(NGPU, 8)
    nbytes = 32 << 20
    outs = run_world(n, list(range(n)), nbytes, 0, 0)
    check_world(oracle, outs, n, nbytes)


def test_nvml_oracle_runs_on_this_box(oracle):
    """The CPU baseline leg itself: real libnvidia-ml.so.1, config 1 (enumerate + NvLinkState poll)."""
    o = oracle.nvml_poll()
    assert o.n >= 1 and o.nvml_calls >= 18 * o.n
    assert all(o.reach[i * 16 + i] == 1 for i in range(o.n))
    assert (o.cc_major[0], o.cc_minor[0]) == (9, 0)


# ------------------------------------------------------ round 2: gate, barriers, abort drain ----
def _cells(n):
    return [(i, j) for i in range(n) for j in range(n) if i != j]


def test_bandwidth_gate_fails_a_slow_but_reachable_domain(pkg, oracle):
    """The bandwidth branch of the verdict (VERDICT r01 weak #4): with a gate nobody can meet every pair is
    reachable yet the verdict is NotReady, counted as slow — not unreachable — pairs; with the gate lowered
    the same handle passes.  Same-device ranks, so it runs on a 1-GPU box."""
    n, nbytes = 3, 4 << 20
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=8, timeout_ms=20000,
                             min_fraction=0.99, link_peak_gbps=1e6)) as p:
        r = p.Run()
        check_full_parity(pkg, oracle, r, n, nbytes, pkg.abi.MODE_SLICED, 3)
        assert r.reach == [[1] * n for _ in range(n)] and not r.aborted
        assert not r.verdict and r.slow_pairs == n * (n - 1) and r.unreachable_pairs == 0
        assert r.gate_gbps_read == pytest.approx(0.99e6, rel=1e-5) and r.gate_gbps_write == pytest.approx(0.99e6, rel=1e-5)
        p.SetOption(pkg.abi.OPT_LINK_PEAK_MBPS, 1)          # 0.001 GB/s x 0.99: everything passes
        r = p.Run()
        assert r.verdict and r.slow_pairs == 0 and r.unreachable_pairs == 0
        # the default reference: 0.65 x bytes_per_pair / (bytes_per_pair / 450 GB/s + 6 us)
        p.SetOption(pkg.abi.OPT_LINK_PEAK_MBPS, 0)
        p.SetOption(pkg.abi.OPT_MIN_FRACTION_PPM, 0)
        r = p.Run()
        bpp = r.bytes_per_pair
        assert r.gate_gbps_read == pytest.approx(0.65 * bpp / (bpp / 450.0 + 6000.0), rel=1e-4)
        assert r.gate_gbps_write == pytest.approx(0.65 * bpp / (bpp / 450.0 + 6000.0), rel=1e-4)


def test_throttled_issuer_fails_only_its_own_pairs(pkg, oracle):
    """A rank whose transfers crawl (1 CTA instead of 8) drags only the pairs IT issues under a gate placed
    between the two speeds; the other ranks' rows stay at speed and the matrices stay all-ones."""
    n, nbytes = 3, 16 << 20
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=8, timeout_ms=20000,
                             min_fraction=1.0, link_peak_gbps=1e-3)) as p:
        p.SetOption(pkg.abi.OPT_CTAS_RANK, (1 << 16) | 1)  # local rank 0 -> one CTA
        assert p.Info().ctas[0] == 1 and p.Info().ctas[1] == 8
        p.Run()
        rs = [p.Run() for _ in range(3)]
        slow = max(max(r.gbps_read[0][j], r.gbps_write[0][j]) for r in rs for j in range(1, n))
        fast = min(min(r.gbps_read[i][j], r.gbps_write[i][j]) for r in rs for i in range(1, n) for j in range(n) if i != j)
        if fast < 1.5 * slow:
            pytest.skip(f"no clean separation on this box (slow {slow:.0f}, fast {fast:.0f} GB/s)")
        thr = (slow * fast) ** 0.5
        p.SetOption(pkg.abi.OPT_LINK_PEAK_MBPS, int(thr * 1e3))
        r = p.Run()
        check_full_parity(pkg, oracle, r, n, nbytes, pkg.abi.MODE_SLICED, 3)
        assert r.reach == [[1] * n for _ in range(n)]
        assert not r.verdict and r.unreachable_pairs == 0 and r.slow_pairs == n - 1  # exactly row 0
        for i, j in _cells(n):
            under = r.gbps_read[i][j] < thr or r.gbps_write[i][j] < thr
            assert under == (i == 0), (i, j, r.gbps_read[i][j], r.gbps_write[i][j], thr)


@pytest.mark.parametrize("n", [2, 4, 5])
def test_barrier_schedules_agree(pkg, oracle, n):
    """The default schedule (neighbourhood exchanges between rounds, NO wait between the write and the read phase of
    a round — the verify job polls for its writer's signal), the same with the pair exchange kept, and round 1's
    all-rank exchange everywhere: same bits, same checksums, run after run."""
    nbytes = 2 << 20
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=8, timeout_ms=20000)) as p:
        for all_rank, pair in ((0, 0), (0, 1), (1, 0), (0, 0)):
            p.SetOption(pkg.abi.OPT_ALL_RANK_BARRIERS, all_rank)
            p.SetOption(pkg.abi.OPT_PAIR_BARRIERS, pair)
            for _ in range(3):
                r = p.Run()
                check_full_parity(pkg, oracle, r, n, nbytes, pkg.abi.MODE_SLICED, 3)
                assert r.reach == [[1] * n for _ in range(n)] and not r.aborted
            tr = p.Trace(0)
            inner = [t for t, nxt in zip(tr, tr[1:]) if t["job0"] == "write" and nxt["job0"] == "read" and t["peer0"] == nxt["peer0"]]
            assert inner
            for t in inner:
                if all_rank:
                    assert t["sync_all"] == 1 and t["post_mask"] == 0
                elif pair:
                    assert bin(t["sync_mask"]).count("1") == 1 and t["post_mask"] == 0
                else:
                    assert t["sync_mask"] == 0 and bin(t["post_mask"]).count("1") == 1
            assert tr[-1]["sync_all"] == 1


def test_abort_in_the_middle_of_a_transfer_drains_and_recovers(pkg, oracle):
    """The device watchdog firing while TMA loads are in flight (VERDICT r01 weak #6): the kernel drains what
    it issued and exits cleanly, the call reports the timeout, and the same handle then runs at parity."""
    n, nbytes = 2, 512 << 20
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=4, timeout_ms=20000)) as p:
        ok = p.Run()
        assert ok.reach == [[1] * n for _ in range(n)]
        assert min(ok.device_ms) > 2.0  # the run is long enough for a 1 ms deadline to land inside a phase
        p.SetOption(pkg.abi.OPT_TIMEOUT_MS, 1)
        r = p.Run(allow_timeout=True)
        assert r.aborted and not r.verdict
        p.SetOption(pkg.abi.OPT_TIMEOUT_MS, 20000)
        for _ in range(2):
            good = p.Run()
            assert not good.aborted
            check_full_parity(pkg, oracle, good, n, nbytes, pkg.abi.MODE_SLICED, 3)


def test_run_never_leaves_the_result_as_it_came_in(pkg):
    """ADVICE r01: cdprobe_run fills the whole result before anything can fail (the daemon writes its verdict
    from it whatever the return code), so garbage in the caller's buffer never survives a call."""
    import ctypes as C

    n, nbytes = 2, 1 << 20
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=8, timeout_ms=20000)) as p:
        out = pkg.abi.ResultT()
        C.memset(C.byref(out), 0xAB, C.sizeof(out))
        assert p.run_raw(out) == pkg.abi.OK and out.n == n and out.verdict in (0, 1)
        assert out.abi == pkg.abi.ABI_VERSION and out.reserved1 == 0 and out.aborted == 0


def test_solo_rank_runs_alone_and_reads_at_parity(pkg, oracle):
    """The profiling mode ncu replays (one self-contained kernel, no cross-GPU barrier): the solo rank's reads
    still carry the oracle's checksums; nobody verifies its writes, so reach_write stays 0."""
    n, nbytes = 2, 8 << 20
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=8, timeout_ms=20000)) as p:
        p.Run()
        p.SetOption(pkg.abi.OPT_SOLO_RANK, 1)
        r = p.Run()
        assert r.launches == 1 and not r.aborted and not r.verdict
        assert r.reach_read[0][1] == 1 and r.reach_write[0][1] == 0
        assert (r.sum_read[0][1], r.xor_read[0][1]) == expected_read(oracle, n, nbytes, 1, 0, 1)
        assert (r.sum_write[0][1], r.xor_write[0][1]) == oracle.write_checksum(SEED, 0, 1, r.run_seq, r.bytes_per_pair // 8)
        p.SetOption(pkg.abi.OPT_SOLO_RANK, 0)
        r = p.Run()
        check_full_parity(pkg, oracle, r, n, nbytes, pkg.abi.MODE_SLICED, 3)


def test_copy_engine_reference_runs_on_the_probe_buffers(pkg, oracle):
    n, nbytes = 2, 64 << 20
    with pkg.Open(pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME, ctas=8, timeout_ms=20000)) as p:
        (ms, gbps), = p.CeCopy([(0, 1)], push=True, reps=3)
        assert ms > 0 and gbps > 10
        both = p.CeCopy([(0, 1), (1, 0)], push=False, reps=3)
        assert len(both) == 2 and all(g > 10 for _, g in both)
        r = p.Run()  # the copies scribbled over landing slots: a probe rewrites them before it verifies
        check_full_parity(pkg, oracle, r, n, nbytes, pkg.abi.MODE_SLICED, 3)


@pytest.mark.skipif(NGPU < 2, reason="needs >= 2 GPUs")
def test_default_gate_passes_healthy_nvlink_and_catches_a_throttled_rank(pkg, oracle):
    """On real peers, 1 GiB per GPU: the default gate (0.65 of nominal NVLink 4) passes,
    a rank throttled to 2 CTAs fails exactly the pairs it issues, and the copy engine gives the ceiling."""
    n = min(NGPU, 8)
    with pkg.Open(pkg.Config(ordinals=list(range(n)), bytes=1 << 30, timeout_ms=20000)) as p:
        p.Run()
        r = p.Run()
        assert r.verdict and r.slow_pairs == 0 and r.unreachable_pairs == 0, (r.min_gbps_read, r.min_gbps_write)
        assert 250 < r.gate_gbps_read < 0.65 * 450 and 250 < r.gate_gbps_write < 0.65 * 450
        assert r.min_gbps_read > r.gate_gbps_read and r.min_gbps_write > r.gate_gbps_write
        p.SetOption(pkg.abi.OPT_CTAS_RANK, (1 << 16) | 2)
        p.Run()
        t = p.Run()
        assert t.reach == [[1] * n for _ in range(n)] and not t.verdict
        assert t.slow_pairs == n - 1 and t.unreachable_pairs == 0
        assert all(t.gbps_read[0][j] < t.gate_gbps_read for j in range(1, n))
        assert all(t.gbps_read[i][j] >= t.gate_gbps_read for i in range(1, n) for j in range(n) if i != j)
        p.SetOption(pkg.abi.OPT_CTAS_RANK, (1 << 16) | 132)
        (ms, uni), = p.CeCopy([(0, 1)], push=True, reps=4)
        bidi = p.CeCopy([(0, 1), (1, 0)], push=True, reps=4)
        assert uni > 300 and min(g for _, g in bidi) > 300


def test_topology_agrees_with_the_oracle_on_the_real_nvml(pkg, oracle):
    """a12 / n2 on the box's own libnvidia-ml.so.1 (not the fake): UUID order, MIG flags, active NVLink
    counts, fabric state and clique id (strict and legacy) equal the oracle's restatement of
    nvlib.go:195-363 / go-nvlib device.go:464-495."""
    for strict, flags in ((True, 0), (False, 1)):
        t = pkg.topology(strict=strict)
        o = oracle.nvml_poll(0, flags | 4)  # no imex-ctl exec: the device + clique walk
        assert t.n == o.n >= 1
        assert [t.uuid[i].value.decode() for i in range(t.n)] == o.uuids()
        assert [t.pci_bus_id[i].value.decode() for i in range(t.n)] == [o.pci_bus_id[i].value.decode() for i in range(o.n)] \
            or all(not o.pci_bus_id[i].value for i in range(o.n))
        assert list(t.mig)[:t.n] == list(o.mig_enabled)[:o.n]
        assert list(t.links_active)[:t.n] == list(o.n_links)[:o.n]
        assert list(t.link_mask)[:t.n] == [sum(1 << l for l in range(18) if o.link_active[i][l]) for i in range(o.n)]
        assert list(t.fabric_state)[:t.n] == list(o.fabric_state)[:o.n]
        assert t.clique_id.decode() == o.clique_id.decode()
        assert bool(t.clique_error) == bool(o.clique_err)
        if t.clique_error:
            assert t.clique_error.decode() == o.clique_err_text.decode()
    # and the CUDA side names the same devices: every probe rank's UUID is one NVML enumerated
    with pkg.Open(pkg.Config(ordinals=None, bytes=1 << 20, mode=pkg.abi.MODE_REACH_ONLY, timeout_ms=20000)) as p:
        info = p.Info()
        nv = set(o.uuids())
        assert all(info.uuid[i].value.decode() in nv for i in range(info.n_local))


# ---- faults: the KERNELS' matrix under an injected fault == the ORACLE's matrix under NVML's statement of it ----
def _oracle_reach_for(tmp_path, scenario, n):
    """The reachability matrix the oracle derives from a (fake) NVML that reports `scenario` (fresh process:
    the fake library reads its script at load; reuses the harness of tests/test_oracle_nvml.py)."""
    from test_oracle_nvml import poll

    r = poll(tmp_path, scenario)
    assert r["rc"] == 0 and r["n"] == n
    return r["reach"]


FAULTS = [
    # (name, NVML scenario, kernel-side injection: list of (local rank, peer) mappings torn down, flags)
    ("healthy", "gpus 4\n", [], 0),
    ("p2p-disabled-pair", "gpus 4\np2p 1 2 nvlink 6\np2p 2 1 nvlink 6\n", [(1, 2)], 0),          # DISABLED_BY_REGKEY, both ways
    ("p2p-read-and-write-off", "gpus 4\np2p 0 3 read 3\np2p 3 0 write 4\n", [(3, 0)], 0),
    ("all-links-down-on-gpu-2", "gpus 4\n" + "".join(f"link_down 2 {l}\n" for l in range(18)), [(2, 0), (2, 1), (2, 3)], 0),
    ("gpu-3-in-mig-mode", "gpus 4\nmig 3 1\n", [(3, 0), (3, 1), (3, 2)], 0),
    ("every-gpu-a-mig-instance", "gpus 4\n" + "".join(f"mig {g} 1\n" for g in range(4)), [], 0x200),  # SIMULATE_MIG
]


@pytest.mark.parametrize("real_peers", [False, True], ids=["same-device", "real-nvlink"])
@pytest.mark.parametrize("name,scenario,unmaps,flags", FAULTS, ids=[f[0] for f in FAULTS])
def test_kernel_matrix_under_faults_equals_oracle_matrix(pkg, oracle, tmp_path, name, scenario, unmaps, flags, real_peers):
    """VERDICT r01 weak #1: the boolean half of parity under faults used to be oracle vs the product's NVML
    walk only.  Here the fault is injected on the DEVICE side (mappings torn down: the loads/stores of that
    pair cannot happen; MIG: no peer mapping at all) and the matrix the kernels produce must equal, bit for
    bit, the matrix the oracle computes from an NVML that reports the same fault (link down on every link of
    a GPU, P2P disabled for a pair, MIG mode).  The kernels treat a pair as one unit — a torn mapping in
    either direction zeroes both cells — so the NVML scenarios state the fault for both ordered pairs."""
    n, nbytes = 4, 1 << 20
    if real_peers and NGPU < n:
        pytest.skip("needs 4 GPUs")
    exp = _oracle_reach_for(tmp_path, scenario, n)
    # same-device: four ranks on GPU 0 (runs on a 1-GPU box); real-nvlink: four GPUs, cooperative launch, one CTA per SM
    cfg = (pkg.Config(ordinals=list(range(n)), bytes=nbytes, flags=flags, timeout_ms=20000) if real_peers else
           pkg.Config(ordinals=[0] * n, bytes=nbytes, flags=SAME | flags, ctas=8, timeout_ms=20000))
    with pkg.Open(cfg) as p:
        for local, peer in unmaps:
            p.UnmapPeer(local, peer)
        r = p.Run()
        assert not r.aborted
        assert r.reach == exp, (name, r.reach, exp)
        healthy = all(all(c == 1 for c in row) for row in exp)
        mig_only = bool(flags & 0x200)
        assert r.verdict == (healthy or mig_only)  # a MIG-only domain is "not applicable", not a failure (SURVEY H8)
        if not mig_only:
            assert r.unreachable_pairs == sum(1 for i in range(n) for j in range(n) if i != j and not exp[i][j])
        # cells that are still reachable carry the oracle's checksums
        for i in range(n):
            for j in range(n):
                if i != j and exp[i][j]:
                    assert (r.sum_read[i][j], r.xor_read[i][j]) == expected_read(oracle, n, nbytes, 1, i, j)
