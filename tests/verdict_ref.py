"""Plain restatement of the probe's verdict arithmetic, written from the field comments of cdprobe_result_t
(include/cdprobe.h) and DESIGN §7 "The verdict gate", not from the library's code.

Given a result, the per-phase trace of every rank whose row it covers, the ops the run judged and whether the plan
has a loop-back slot, `expected()` says what `unreachable_pairs`, `slow_pairs`, `min_gbps_read`, `min_gbps_write`
and `verdict` must be:

- A cell (issuer i, target j) of an op is *filled* when a phase of i's trace has job 0 = that op with peer j.  The
  min rate is taken over filled off-diagonal cells, or over the diagonal when n == 1; 0 when there are none.
- A cell whose status, or its transpose's, is ERR_UNSUPPORTED (a MIG instance has no peer) counts toward neither the
  pair counts nor the verdict.
- An off-diagonal cell is unreachable when an op in `ops` has reach 0; it is slow when it is reachable and one of
  its rates of an op in `ops` is under that op's gate (a strict float32 `<`).  Unreachable takes precedence: a cell
  is counted once, in one of the two.
- The loop-back cell gates the verdict only when n == 1, and only by reachability.
- An aborted run has verdict 0.

The result is duck-typed: a fabricprobe.Result, or anything with the same attribute names (the CPU tests build them
by hand, the two-process tests rebuild them from JSON).  Traces are what `Probe.Trace()` returns, keyed by global
rank.
"""
from __future__ import annotations

import numpy as np

OP_READ, OP_WRITE = 1, 2
ERR_UNSUPPORTED = -8
OPS = ((OP_READ, "read"), (OP_WRITE, "write"))


def rows(res):
    return [i for i in range(res.n) if (res.row_mask >> i) & 1]


def filled_cells(traces, op_name):
    """{(issuer, target)} of the cells whose rate a phase of the issuer's trace carries (job 0 only)."""
    return {(i, ph["peer0"]) for i, tr in traces.items() for ph in tr if ph["job0"] == op_name}


def mig_excluded(res, i, j):
    return res.status[i][j] == ERR_UNSUPPORTED or res.status[j][i] == ERR_UNSUPPORTED


def expected(res, traces, ops, loopback):
    """What the verdict fields of `res` must be.  `traces` maps every row of res.row_mask to its trace; `ops` is the
    config's ops (0 = read | write); `loopback` says whether the plan has a diagonal slot (n == 1 or LOCAL_DIAG)."""
    assert set(traces) == set(rows(res)), (sorted(traces), res.row_mask)
    ops = ops or (OP_READ | OP_WRITE)
    n = res.n
    gate = {"read": np.float32(res.gate_gbps_read), "write": np.float32(res.gate_gbps_write)}
    reach = {"read": res.reach_read, "write": res.reach_write}
    gbps = {"read": res.gbps_read, "write": res.gbps_write}

    mins = {}
    for _, name in OPS:
        cells = [(i, j) for i, j in filled_cells(traces, name) if i != j or n == 1]
        mins[name] = float(min((np.float32(gbps[name][i][j]) for i, j in cells), default=np.float32(0.0)))

    judged = [(bit, name) for bit, name in OPS if ops & bit]
    unreachable = slow = 0
    verdict = True
    for i in rows(res):
        for j in range(n):
            if i == j or mig_excluded(res, i, j):
                continue
            if any(not reach[name][i][j] for _, name in judged):
                unreachable += 1
                verdict = False
            elif any(np.float32(gbps[name][i][j]) < gate[name] for _, name in judged):
                slow += 1
                verdict = False
        if n == 1 and loopback and any(not reach[name][i][i] for _, name in judged):
            verdict = False
    if res.aborted:
        verdict = False
    return {"unreachable_pairs": unreachable, "slow_pairs": slow, "min_gbps_read": mins["read"],
            "min_gbps_write": mins["write"], "verdict": verdict}


def check(res, traces, ops, loopback, gate):
    """Assert that `res` carries the verdict the restatement gives, and that it applied `gate` = (read, write), the
    GB/s threshold `cdprobe_gate` states for its config and rank count.  Returns the expectation."""
    assert (np.float32(res.gate_gbps_read), np.float32(res.gate_gbps_write)) == tuple(np.float32(g) for g in gate), \
        ((res.gate_gbps_read, res.gate_gbps_write), gate)
    want = expected(res, traces, ops, loopback)
    got = {"unreachable_pairs": res.unreachable_pairs, "slow_pairs": res.slow_pairs,
           "min_gbps_read": float(np.float32(res.min_gbps_read)), "min_gbps_write": float(np.float32(res.min_gbps_write)),
           "verdict": bool(res.verdict)}
    assert got == want, {"got": got, "want": want}
    return want
