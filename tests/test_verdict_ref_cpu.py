"""The verdict restatement (tests/verdict_ref.py) pinned on hand-built results, one rule per test, so that the
reference is itself tested before tests/test_timing_gpu.py uses it to judge the library."""
import types

import numpy as np
import pytest

import verdict_ref as ref

GATE = 100.0  # GB/s, read and write, for every hand-built result below
FAST = 200.0
MIG = ref.ERR_UNSUPPORTED


def make(n, gbps=FAST, reach=1, diag=False, ops=3, gate=GATE, aborted=False):
    """A healthy-looking result over n ranks in one process: every off-diagonal cell (and the diagonal when `diag`)
    filled by one read and one write phase at `gbps`, all reachable; the verdict fields are left for the test."""
    cells = [(i, j) for i in range(n) for j in range(n) if i != j or diag]
    res = types.SimpleNamespace(
        n=n, row_mask=(1 << n) - 1, aborted=aborted, gate_gbps_read=gate, gate_gbps_write=gate,
        reach_read=[[1] * n for _ in range(n)], reach_write=[[1] * n for _ in range(n)],
        gbps_read=[[0.0] * n for _ in range(n)], gbps_write=[[0.0] * n for _ in range(n)],
        status=[[0] * n for _ in range(n)])
    traces = {i: [] for i in range(n)}
    for i, j in cells:
        for bit, name in ref.OPS:
            if ops & bit:
                getattr(res, "gbps_" + name)[i][j] = gbps
                getattr(res, "reach_" + name)[i][j] = reach
                traces[i].append({"job0": name, "peer0": j})
    return res, traces


def test_min_is_over_filled_off_diagonal_cells():
    res, traces = make(3)
    res.gbps_read[0][1] = 150.0
    res.gbps_write[2][0] = 120.0
    res.gbps_read[1][1] = 5.0   # not filled: no phase of rank 1 reads itself
    want = ref.expected(res, traces, 3, loopback=False)
    assert (want["min_gbps_read"], want["min_gbps_write"]) == (150.0, 120.0)
    traces[1].append({"job0": "read", "peer0": 1})  # filled, but on the diagonal of a 3-rank domain
    assert ref.expected(res, traces, 3, loopback=True)["min_gbps_read"] == 150.0
    traces[1].append({"job0": "verify", "peer0": 2})  # a verify carries no rate
    res.gbps_write[1][2] = 1.0
    assert ref.expected(res, traces, 3, loopback=True)["min_gbps_write"] == 1.0  # (1, 2) is filled by its write


def test_min_is_the_diagonal_at_one_rank_and_zero_without_cells():
    res, traces = make(1, gbps=3000.0, diag=True, gate=0.0)
    res.gbps_write[0][0] = 2500.0
    want = ref.expected(res, traces, 3, loopback=True)
    assert (want["min_gbps_read"], want["min_gbps_write"], want["verdict"]) == (3000.0, 2500.0, True)
    res, traces = make(2, ops=1)
    want = ref.expected(res, traces, 1, loopback=False)
    assert (want["min_gbps_read"], want["min_gbps_write"]) == (FAST, 0.0)


def test_mig_cells_count_toward_nothing():
    res, traces = make(3)
    for i, j in ((0, 1), (1, 0)):
        res.status[i][j] = MIG
        res.reach_read[i][j] = res.reach_write[i][j] = 0
    want = ref.expected(res, traces, 3, loopback=False)
    assert (want["unreachable_pairs"], want["slow_pairs"], want["verdict"]) == (0, 0, True)
    res.status[1][0] = 0  # the transpose alone excludes the cell too
    assert ref.expected(res, traces, 3, loopback=False)["unreachable_pairs"] == 0


def test_unreachable_needs_an_op_in_ops():
    res, traces = make(3)
    res.reach_write[0][2] = 0
    assert ref.expected(res, traces, 3, loopback=False)["unreachable_pairs"] == 1
    assert ref.expected(res, traces, 1, loopback=False) == {
        "unreachable_pairs": 0, "slow_pairs": 0, "min_gbps_read": FAST, "min_gbps_write": FAST, "verdict": True}


def test_slow_is_a_strict_float32_comparison_counted_per_cell():
    gate = float(np.float32(123.456))
    res, traces = make(2, gate=gate)
    res.gbps_read[0][1] = gate  # equal: at speed
    assert ref.expected(res, traces, 3, loopback=False)["slow_pairs"] == 0
    below = float(np.nextafter(np.float32(gate), np.float32(0)))
    res.gbps_read[0][1] = below
    res.gbps_write[0][1] = below  # both ops under the gate: still one cell
    want = ref.expected(res, traces, 3, loopback=False)
    assert (want["slow_pairs"], want["unreachable_pairs"], want["verdict"]) == (1, 0, False)
    assert ref.expected(res, traces, 2, loopback=False)["slow_pairs"] == 1  # the write alone is judged
    res.gbps_write[0][1] = FAST
    assert ref.expected(res, traces, 2, loopback=False)["slow_pairs"] == 0  # an op outside ops is not judged


def test_unreachable_takes_precedence_over_slow():
    res, traces = make(4, gbps=1.0)  # every cell under the gate
    res.reach_read[2][0] = 0
    want = ref.expected(res, traces, 3, loopback=False)
    assert (want["unreachable_pairs"], want["slow_pairs"], want["verdict"]) == (1, 11, False)


def test_loopback_gates_only_at_one_rank_and_only_by_reach():
    res, traces = make(1, diag=True, gbps=1.0, gate=5.0)  # under a (hypothetical) gate: not judged
    assert ref.expected(res, traces, 3, loopback=True)["verdict"] is True
    res.reach_read[0][0] = 0
    want = ref.expected(res, traces, 3, loopback=True)
    assert (want["verdict"], want["unreachable_pairs"]) == (False, 0)
    assert ref.expected(res, traces, 2, loopback=True)["verdict"] is True  # the read is not judged
    res, traces = make(4, diag=True)
    res.reach_write[3][3] = 0
    res.gbps_read[1][1] = 1.0
    want = ref.expected(res, traces, 3, loopback=True)
    assert (want["verdict"], want["slow_pairs"], want["min_gbps_read"]) == (True, 0, FAST)


def test_aborted_forces_verdict_zero():
    res, traces = make(2, aborted=True)
    want = ref.expected(res, traces, 3, loopback=False)
    assert (want["verdict"], want["unreachable_pairs"], want["slow_pairs"]) == (False, 0, 0)


def test_only_the_rows_of_the_result_are_judged():
    res, traces = make(3)
    res.row_mask = 0b010
    res.reach_read[0][1] = 0  # row 0 belongs to another process
    res.gbps_write[1][2] = 150.0
    del traces[0], traces[2]
    want = ref.expected(res, traces, 3, loopback=False)
    assert (want["unreachable_pairs"], want["verdict"], want["min_gbps_write"]) == (0, True, 150.0)
    with pytest.raises(AssertionError):
        ref.expected(res, {0: [], 1: []}, 3, loopback=False)  # a trace per row, no more, no less


def test_check_compares_every_field_and_the_gate():
    res, traces = make(2)
    res.gbps_read[1][0] = 1.0
    res.unreachable_pairs, res.slow_pairs, res.verdict = 0, 1, 0
    res.min_gbps_read, res.min_gbps_write = 1.0, FAST
    ref.check(res, traces, 3, False, (GATE, GATE))
    with pytest.raises(AssertionError):
        ref.check(res, traces, 3, False, (GATE, GATE * 2))  # the gate the config states is not the one applied
    for field, bad in (("slow_pairs", 2), ("unreachable_pairs", 1), ("min_gbps_read", 2.0), ("verdict", 1)):
        good = getattr(res, field)
        setattr(res, field, bad)
        with pytest.raises(AssertionError):
            ref.check(res, traces, 3, False, (GATE, GATE))
        setattr(res, field, good)
