"""A catalogue of deliberate one-place errors in the sources of libcdprobe.so, each of which a named GPU test must see.

Every entry (MUTANTS) names a source file under k8s-dra-driver-gpu_b200/csrc/, the function (or struct) whose body
holds the change, an anchor text that occurs exactly once in that body, its replacement and the GPU tests expected to
fail with the change (killers); KILLED_BY records the test that did fail when tools/mutants.py last ran the catalogue
on an H100 (the first failing test of one `pytest -m gpu -x` over the killers).  test_mutants_cpu.py checks every entry
on the CPU: the anchor applies once inside its function, the mutated unit compiles for sm_90a, every killer exists.

A mutant changes only a value that is computed, stored or compared (safety_problems enforces what it can of that):
never an address or offset, a loop bound, unit count or walk, a flag, epoch or wait target, a fence, a barrier or a
deadline.  So every access stays inside its allocation and every wait stays satisfiable, and a mutant can make a
kernel report a wrong result but cannot fault it or hang it.

Changes that no test can observe are not in the table; what they were, and why they are invisible:
  * an xor of a constant into every warp's X part (bwcurve_kernel's Sum): a grid has 8 warps per CTA, an even count,
    so the constants cancel in the CTA and grid reductions;
  * the pingpong initiator's `v != ping + 1` status check: a wrong echo also changes the rep's digest, which the host
    compares with the clean digest, so the cell is CDPROBE_ERR_INTEGRITY either way;
  * the atomics chain's per-op `bad` test: an op that returns a wrong value leaves the word, which is read back, and
    the digest wrong as well;
  * in job_read_tma, swapping the high halves of a vector's two words (pack64(v.x, v.w), pack64(v.z, v.y)): S adds
    the two words and X xors them, so both are unchanged;
  * fold_checks comparing the warm-up copy's (S, X) with want no more: a landed word that differs from the pattern
    also counts in the rep's bad words, which fold_checks adds over every rep, warm-up included, and a check whose
    (S, X) fold were wrong would be wrong in the timed reps too."""
import difflib
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "k8s-dra-driver-gpu_b200", "csrc")


def replace_once(text, old, new, where="the text"):
    """text with the one occurrence of old replaced by new; fails loudly when old occurs other than once."""
    n = text.count(old)
    assert n == 1, f"{old!r} occurs {n} times in {where}"
    return text.replace(old, new)


def _blank(text):
    """text with every comment and the inside of every string and character literal replaced by spaces, offsets kept."""
    out = list(text)
    for m in re.finditer(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'', text, re.S):
        for i in range(m.start() + (m.group()[0] in "\"'"), m.end() - (m.group()[0] in "\"'")):
            if out[i] != "\n":
                out[i] = " "
    return "".join(out)


def _close(code, i, open_c, close_c):
    """Index just past the bracket that closes the one at code[i]."""
    depth = 0
    for j in range(i, len(code)):
        if code[j] == open_c:
            depth += 1
        elif code[j] == close_c:
            depth -= 1
            if depth == 0:
                return j + 1
    raise AssertionError(f"unbalanced {open_c} at offset {i}")


def body(text, function):
    """(start, end) offsets of the body of the one definition of `function` (a function or a struct) in text, braces
    included.  A definition is `struct NAME ... {` or `NAME(params) qualifiers {`; calls, declarations and braced
    initialisers are not."""
    code = _blank(text)
    spans = []
    name = re.escape(function)
    for m in re.finditer(r"\bstruct\s+" + name + r"\b[^;{()]*\{", code):
        spans.append((m.end() - 1, _close(code, m.end() - 1, "{", "}")))
    for m in re.finditer(r"(?<![\w.>:])" + name + r"\s*\(", code):
        end = _close(code, m.end() - 1, "(", ")")
        tail = re.match(r"[^;{}()=,]*\{", code[end:])
        if tail:
            start = end + tail.end() - 1
            spans.append((start, _close(code, start, "{", "}")))
    assert len(spans) == 1, f"{function}: {len(spans)} definitions found"
    return spans[0]


def apply(text, m):
    """text (the source of m['file']) with mutant m applied: its anchor replaced, once, inside its function's body."""
    start, end = body(text, m["function"])
    return text[:start] + replace_once(text[start:end], m["old"], m["new"], f"{m['function']} of {m['file']}") + \
        text[end:]


def mutated(m, root=ROOT):
    """The source of m's file under root's csrc/ with m applied."""
    with open(os.path.join(root, "k8s-dra-driver-gpu_b200", "csrc", m["file"])) as f:
        return apply(f.read(), m)


# ---- the safety rule ------------------------------------------------------------------------------------------------
# Names a mutant may not add, remove or change: control flow, waits, flags, fences, barriers, deadlines, walks and
# unit counts.
FORBIDDEN = {
    "for", "while", "do", "break", "continue", "return", "goto", "take", "Walk", "BlockWalk", "strided", "claimed",
    "units_of", "unit_len", "n_units", "units", "lines", "words", "len", "nvec", "bytes", "nwarps", "gwarp", "span",
    "reps", "n_sizes", "ops", "hops", "trips", "spin_until", "mbar_wait", "mbar_drain", "mbar_try_wait", "wait_flag",
    "poll", "ld_flag", "st_flag", "flag", "f0", "f1", "ll_flag", "ring_flag", "handover", "signal", "signal_ranks",
    "grid_barrier", "close_fenced", "barrier", "__syncthreads", "__syncthreads_or", "__syncwarp", "__threadfence",
    "__threadfence_system", "fence_proxy_async_global", "fence_proxy_async_smem", "fence_proxy_alias",
    "bulk_wait_read", "bulk_wait_all", "bulk_commit", "deadline", "timeout_ns", "check_abort", "aborted", "abort_word",
    "abort_flag", "release", "arrive", "call_seq", "seq_base", "written", "claim", "done", "target", "__trap",
}
# Calls whose first argument is an address: it must stay as it is, and no such call may be added or removed.
ADDRESS_CALLS = {
    "stg_v4", "stg_pair", "sts_v4", "lds_v4", "ldg_stream_v4", "ldg_nc_v4", "__ldcg", "__ldg", "st_relaxed_sys",
    "ld_relaxed_sys", "st_release_sys", "st_release_gpu", "ld_acquire", "st_packet", "ld_packet", "red_add_sys",
    "bulk_load", "bulk_store", "bulk_reduce_add_u64", "issue_load", "sts_u64", "lds_u64", "mc_ld_reduce_add_u64",
    "mc_st_v4", "atom_exch", "atom_add", "atom_cas", "atomicAdd", "atomicMax", "atomicXor", "atomicExch", "xor_landing",
}


def _tokens(text):
    return re.findall(r"\w+|\S", text)


def _address_args(text):
    """Sorted (call, first argument) of every address-taking call in text."""
    out = []
    for m in re.finditer(r"\b(" + "|".join(sorted(ADDRESS_CALLS)) + r")\s*(<[^<>()]*>)?\s*\(", text):
        i, depth = m.end(), 0
        for j in range(i, len(text)):
            if text[j] in "([{":
                depth += 1
            elif text[j] in ")]}":
                if depth == 0:
                    break
                depth -= 1
            elif text[j] == "," and depth == 0:
                break
        out.append((m.group(1), " ".join(text[i:j].split())))
    return sorted(out)


def _in_loop_header(tokens, i1, i2):
    """Whether tokens[i1:i2] (or the insertion point i1) lies inside the parentheses of a for or while."""
    for i in range(i1, max(i1 + 1, i2)):
        depth = 0
        for j in range(min(i, len(tokens)) - 1, -1, -1):
            if tokens[j] == ")":
                depth += 1
            elif tokens[j] == "(":
                if depth == 0 and j > 0 and tokens[j - 1] in ("for", "while"):
                    return True
                depth = max(0, depth - 1)
    return False


def safety_problems(m):
    """What in mutant m breaks the safety rule (empty when nothing does): a forbidden name among the tokens it changes,
    a subscript it adds or removes, or an address-taking call whose address it changes, adds or removes."""
    problems = []
    a, b = _tokens(m["old"]), _tokens(m["new"])
    changed = set()
    for op, i1, i2, j1, j2 in difflib.SequenceMatcher(a=a, b=b, autojunk=False).get_opcodes():
        if op != "equal":
            changed.update(a[i1:i2] + b[j1:j2])
            if _in_loop_header(a, i1, i2) or _in_loop_header(b, j1, j2):
                problems.append("changes a loop header")
    bad = sorted(changed & FORBIDDEN)
    if bad:
        problems.append(f"changes {bad}")
    subs = [set(" ".join(s.split()) for s in re.findall(r"\[([^\[\]]*)\]", t)) for t in (m["old"], m["new"])]
    if subs[0] != subs[1]:
        problems.append(f"subscripts {sorted(subs[0] ^ subs[1])}")
    if _address_args(m["old"]) != _address_args(m["new"]):
        problems.append(f"addresses {_address_args(m['old'])} -> {_address_args(m['new'])}")
    return problems


# ---- the catalogue --------------------------------------------------------------------------------------------------
# The first failing test of each mutant when tools/mutants.py last ran the catalogue (NVIDIA H100 80GB HBM3, 700 W).
KILLED_BY = {
    "pattern_lane_swap": "tests/test_words_gpu.py::test_loopback_regions_every_path_and_tail[128]",
    "fold_unit_neighbour_granule": "tests/test_gpu_parity.py::test_single_gpu_small_sizes[128-tma]",
    "add_pair_drops_w1_from_x": "tests/test_gpu_parity.py::test_single_gpu_small_sizes[128-tma]",
    "granule_sum_adds_x": "tests/test_bwcurve_gpu.py::test_loopback_every_size_clean[4MiB-tma]",
    "verdict_ignores_x": "tests/test_landing_faults_gpu.py::test_write_checksum_blind_spot_on_the_device",
    "row_expected_source_sum_off": "tests/test_gpu_parity.py::test_single_gpu_small_sizes[128-tma]",
    "fill_src_odd_word_from_even": "tests/test_gpu_parity.py::test_single_gpu_small_sizes[128-tma]",
    "loopback_last_stamp_late": "tests/test_timing_gpu.py::test_single_gpu_stamps_events_and_verdict[128B-tma]",
    "diag_last_bad_one_word_late": "tests/test_diagnose_gpu.py::test_flipped_bits_are_counted_located_and_sampled",
    "diag_sample_observed_flipped": "tests/test_diagnose_gpu.py::test_flipped_bits_are_counted_located_and_sampled",
    "diag_high_flips_counted_once": "tests/test_words_gpu.py::test_a_granule_with_every_word_flipped",
    "latency_first_hop_digest_off": "tests/test_latency_gpu.py::test_loopback_chase_digest_and_times[128B]",
    "latency_warmup_digest_dropped": "tests/test_latency_gpu.py::test_loopback_chase_digest_and_times[1MiB]",
    "tma_partial_unit_halves_swapped": "tests/test_gpu_parity.py::test_single_gpu_small_sizes[128-tma]",
    "latency_rep_time_plus_100us": "tests/test_timing_gpu.py::test_latency_per_hop",
    "atomics_chain_digest_adds": "tests/test_atomics_gpu.py::test_every_cell_clean[n1-fetch_add]",
    "atomics_chain_rep_time_plus_100us": "tests/test_timing_gpu.py::test_atomics_per_op[fetch_add]",
    "bwcurve_warmup_sum_off": "tests/test_bwcurve_gpu.py::test_loopback_every_size_clean[4MiB-tma]",
    "bwcurve_first_timed_rep_sum_off": "tests/test_bwcurve_gpu.py::test_loopback_every_size_clean[4MiB-tma]",
    "a2a_check_fold_by_unit": "tests/test_alltoall_gpu.py::test_single_rank_every_size_clean[4MiB-tma]",
    "a2a_salt_sender_receiver_swapped": "tests/test_alltoall_gpu.py::test_same_device_every_cell_clean[2-sliced]",
    "oneshot_fault_halves_swapped": "tests/test_allreduce_gpu.py::test_an_armed_fault_fails_exactly_one_row_and_size",
    "oneshot_fault_every_timed_rep": "tests/test_allreduce_gpu.py::test_an_armed_fault_fails_exactly_one_row_and_size",
    "oneshot_full_unit_words_swapped": "tests/test_allreduce_gpu.py::test_single_rank_every_size_clean[4MiB-tma]",
    "twoshot_fault_on_neighbour_word": "tests/test_allreduce_twoshot_gpu.py::test_grids_and_faults_at_the_edges[ctas1]",
    "ll_last_word_off": "tests/test_allreduce_ll_gpu.py::test_tiny_ladders_and_the_ladder_cut_at_1_mib[1-128]",
    "ll_x_folded_per_line": "tests/test_allreduce_ll_gpu.py::test_tiny_ladders_and_the_ladder_cut_at_1_mib[1-4096]",
    "diag_single_bad_granule_uncounted":
        "tests/test_diagnose_gpu.py::test_flipped_bits_are_counted_located_and_sampled",
    "a2a_first_bad_odd_word_late":
        "tests/test_alltoall_gpu.py::test_an_armed_fault_fails_exactly_its_cell_and_size[tma]",
    "twoshot_drop_mode_ignored":
        "tests/test_allreduce_twoshot_gpu.py::test_a_dropped_unit_reads_as_zeros_because_every_rep_clears_the_output",
    "ll_fault_to_every_other_peer":
        "tests/test_allreduce_ll_gpu.py::test_a_corrupted_packet_fails_only_its_receiver_and_size",
    "ring_own_store_words_swapped": "tests/test_allreduce_ring_gpu.py::test_single_rank_every_size_clean[4MiB]",
    "ring_fault_in_the_other_phase":
        "tests/test_allreduce_ring_gpu.py::test_a_faulted_push_fails_exactly_the_rows_the_restatement_names[corrupt]",
    "ring_fault_halves_swapped":
        "tests/test_allreduce_ring_gpu.py::test_a_faulted_push_fails_exactly_the_rows_the_restatement_names[corrupt]",
    "push_ldst_fault_halves_swapped":
        "tests/test_allreduce_push_gpu.py::test_each_fault_fails_exactly_the_rows_and_words_the_restatement_names[1-1]",
    "push_mode_2_disarmed":
        "tests/test_allreduce_push_gpu.py::test_each_fault_fails_exactly_the_rows_and_words_the_restatement_names[1-0]",
    "push_gather_fault_one_word_late":
        "tests/test_allreduce_push_gpu.py::test_each_fault_fails_exactly_the_rows_and_words_the_restatement_names[2-0]",
    "nvls_vector_words_swapped": "tests/test_allreduce_nvls_emulated_gpu.py::test_clean_ladders_on_every_grid[1-128]",
    "nvls_fault_on_every_other_vector":
        "tests/test_allreduce_nvls_emulated_gpu.py::"
        "test_each_fault_fails_exactly_the_words_the_restatement_names[1-467328-2]",
    "nvls_fault_in_the_warmup":
        "tests/test_allreduce_nvls_emulated_gpu.py::"
        "test_each_fault_fails_exactly_the_words_the_restatement_names[1-467328-2]",
    "ar_add_low_carry_lost": "tests/test_allreduce_gpu.py::test_same_device_every_row_clean[2-sliced]",
    "ar_check_clear_stores_the_word_back":
        "tests/test_allreduce_gpu.py::test_a_dropped_unit_is_seen_whatever_the_output_held_before",
    "ar_check_clear_first_one_word_late":
        "tests/test_allreduce_gpu.py::test_an_armed_fault_fails_exactly_one_row_and_size",
    "ar_check_stores_the_sum_back":
        "tests/test_allreduce_ll_gpu.py::test_an_unstored_word_is_seen_whatever_the_output_held_before",
    "put_ranks_fault_to_the_next_rank":
        "tests/test_allreduce_twoshot_gpu.py::test_grids_and_faults_at_the_edges[ctas1]",
    "closing_timer_read_100us_late": "tests/test_timing_gpu.py::test_latency_per_hop",
    "closing_timer_read_before_the_opening": "tests/test_timing_gpu.py::test_latency_per_hop",
    "fold_checks_last_rep_only":
        "tests/test_memcpy_gpu.py::test_an_armed_fault_fails_exactly_its_cell_and_size[flip-pull]",
    "fold_checks_first_one_word_late":
        "tests/test_memcpy_gpu.py::test_an_armed_fault_fails_exactly_its_cell_and_size[flip-pull]",
    "summarize_warmup_digest_dropped": "tests/test_latency_gpu.py::test_loopback_chase_digest_and_times[1MiB]",
    "ladder_t0_from_the_minimum": "tests/test_ladder_timing_gpu.py::test_windows_fit_in_the_call[1]",
    "word_checks_first_one_word_late":
        "tests/test_allreduce_gpu.py::test_an_armed_fault_fails_exactly_one_row_and_size",
    "pingpong_digest_of_the_ping":
        "tests/test_rep_records_gpu.py::test_pingpong_digest_over_an_odd_number_of_trips[plain-1]",
    "pingpong_warmup_digest_dropped":
        "tests/test_rep_records_gpu.py::test_pingpong_digest_over_an_odd_number_of_trips[plain-1]",
    "pingpong_rep_time_plus_100us": "tests/test_rep_records_gpu.py::test_short_pingpong_reps_are_not_padded",
    "atomics_contended_digest_sums":
        "tests/test_rep_records_gpu.py::test_atomics_digest_over_an_odd_number_of_ops[contended-1]",
    "bwcurve_rep_end_late": "tests/test_rep_records_gpu.py::test_short_bwcurve_reps_are_not_padded",
    "twoshot_fault_every_timed_rep": "tests/test_rep_records_gpu.py::test_twoshot_fault_acts_in_timed_rep_1_of_3_only",
}


def _m(name, file, function, old, new, killers, why):
    return {"name": name, "file": file, "function": function, "old": old, "new": new, "killers": killers,
            "killed_by": KILLED_BY.get(name), "why": why}


T = "tests/"
WORDS = T + "test_words_gpu.py::"
PARITY = T + "test_gpu_parity.py::"
LANDING = T + "test_landing_faults_gpu.py::"
TIMING = T + "test_timing_gpu.py::"
LADDER_TIMING = T + "test_ladder_timing_gpu.py::"
DIAG = T + "test_diagnose_gpu.py::"
LAT = T + "test_latency_gpu.py::"
PP = T + "test_pingpong_gpu.py::"
AT = T + "test_atomics_gpu.py::"
BW = T + "test_bwcurve_gpu.py::"
A2A = T + "test_alltoall_gpu.py::"
AR = T + "test_allreduce_gpu.py::"
AR2 = T + "test_allreduce_twoshot_gpu.py::"
LL = T + "test_allreduce_ll_gpu.py::"
RING = T + "test_allreduce_ring_gpu.py::"
PUSH = T + "test_allreduce_push_gpu.py::"
NVLS = T + "test_allreduce_nvls_emulated_gpu.py::"
MC = T + "test_memcpy_gpu.py::"
EDGES = T + "test_ladder_edges_gpu.py::"
RR = T + "test_rep_records_gpu.py::"  # the tests added for the mutants nothing else killed

MUTANTS = [
    # ---- datapath.cuh ----
    _m("pattern_lane_swap", "datapath.cuh", "Pattern",
       "2ull * kV * lane) * kGolden) {}", "2ull * kV * (lane ^ 1)) * kGolden) {}",
       [WORDS + "test_loopback_regions_every_path_and_tail", A2A + "test_single_rank_every_size_clean"],
       "lanes 2i and 2i + 1 store each other's runs of the write pattern: the same words in each unit, so (S, X) "
       "cannot see it"),
    _m("fold_unit_neighbour_granule", "datapath.cuh", "fold_unit",
       "rotl64(unit_xor, fold6(g))", "rotl64(unit_xor, fold6(g ^ 1))",
       [PARITY + "test_single_gpu_small_sizes", BW + "test_loopback_every_size_clean"],
       "every unit's xor is rotated by its neighbouring granule's amount"),
    _m("add_pair_drops_w1_from_x", "datapath.cuh", "add_pair",
       "ux ^= w0 ^ w1;", "ux ^= w0;",
       [PARITY + "test_single_gpu_small_sizes", BW + "test_loopback_every_size_clean"],
       "the odd words never reach X"),
    _m("tma_partial_unit_halves_swapped", "datapath.cuh", "job_read_tma",
       "lds_v4(c.stage_smem + s * kUnitBytes + i * 16u);\n        add_pair(a, ux, pack64(v.x, v.y), pack64(v.z, v.w));",
       "lds_v4(c.stage_smem + s * kUnitBytes + i * 16u);\n        add_pair(a, ux, pack64(v.y, v.x), pack64(v.z, v.w));",
       [PARITY + "test_single_gpu_small_sizes", BW + "test_loopback_every_size_clean"],
       "the TMA read of a partial last unit swaps the 32-bit halves of every even word"),
    _m("granule_sum_adds_x", "datapath.cuh", "granules_kernel",
       "x ^= w;", "x += w;",
       [BW + "test_loopback_every_size_clean", AR + "test_single_rank_every_size_clean"],
       "the expected per-granule X, folded into the ladder measurements' want, is a sum"),
    # ---- probe_kernels.cu ----
    _m("verdict_ignores_x", "probe_kernels.cu", "publish_verdicts",
       "(wsum == acc->sum && wxr == acc->xr)", "(wsum == acc->sum)",
       [LANDING + "test_write_checksum_blind_spot_on_the_device", LANDING + "test_every_kind_in_one_write_cell"],
       "the write verdict compares S only"),
    _m("row_expected_source_sum_off", "probe_kernels.cu", "write_row",
       "o.exp_sum[jb] = ld_relaxed_sys(&pc->src_sum[slice]);",
       "o.exp_sum[jb] = ld_relaxed_sys(&pc->src_sum[slice]) + 1;",
       [PARITY + "test_single_gpu_small_sizes", PARITY + "test_same_device_ranks"],
       "the row's expected source S of a read job is one too large"),
    _m("fill_src_odd_word_from_even", "probe_kernels.cu", "cdprobe_fill_src_kernel",
       "w1 = src_word(seed, rank, 2 * v + 1);", "w1 = src_word(seed, rank, 2 * v);",
       [PARITY + "test_single_gpu_small_sizes", WORDS + "test_loopback_regions_every_path_and_tail"],
       "every odd source word repeats the even word before it; the probe's own checks agree with themselves"),
    _m("loopback_last_stamp_late", "probe_kernels.cu", "loopback_pass",
       "ctrl->t_arr[2] = gtimer();", "ctrl->t_arr[2] = gtimer() + 1000000;",
       [TIMING + "test_single_gpu_stamps_events_and_verdict"],
       "the loop-back pass's closing stamp is 1 ms late"),
    # ---- diagnose_kernels.cu ----
    _m("diag_last_bad_one_word_late", "diagnose_kernels.cu", "diag_compare_kernel",
       "atomicMax(&out->last_bad, last * 8ull);", "atomicMax(&out->last_bad, last * 8ull + 8);",
       [DIAG + "test_flipped_bits_are_counted_located_and_sampled", WORDS + "test_diagnosis_equals_the_reference"],
       "last_bad names the word after the last bad one"),
    _m("diag_sample_observed_flipped", "diagnose_kernels.cu", "diag_sample_kernel",
       "o.observed = w[h];", "o.observed = w[h] ^ 1ull;",
       [DIAG + "test_flipped_bits_are_counted_located_and_sampled", WORDS + "test_diagnosis_equals_the_reference"],
       "every sample reports an observed word with bit 0 flipped"),
    _m("diag_high_flips_counted_once", "diagnose_kernels.cu", "diag_compare_kernel",
       "if (lane == (uint32_t)bit) flips_hi += n;", "if (lane == (uint32_t)bit) flips_hi += 1;",
       [WORDS + "test_a_granule_with_every_word_flipped", DIAG + "test_flipped_bits_are_counted_located_and_sampled"],
       "a high bit flipped in several words of one batch row counts once"),
    _m("diag_single_bad_granule_uncounted", "diagnose_kernels.cu", "diag_compare_kernel",
       "granules += gb != 0;", "granules += gb > 1;",
       [DIAG + "test_flipped_bits_are_counted_located_and_sampled", WORDS + "test_diagnosis_equals_the_reference"],
       "a granule with one bad word is not counted in bad_granules"),
    # ---- latency_kernels.cu ----
    _m("latency_first_hop_digest_off", "latency_kernels.cu", "latency_kernel",
       "digest ^= v;", "digest ^= h == 0 ? v + 1 : v;",
       [LAT + "test_loopback_chase_digest_and_times"], "the first hop's word enters the digest plus one"),
    _m("latency_warmup_digest_dropped", "latency_kernels.cu", "latency_kernel",
       "o[r].digest = digest;", "o[r].digest = r == 0 ? 0ull : digest;",
       [LAT + "test_loopback_chase_digest_and_times"], "the warm-up rep's digest is left out"),
    _m("latency_rep_time_plus_100us", "latency_kernels.cu", "latency_kernel",
       "o[r].ns = t1 - t0;", "o[r].ns = t1 - t0 + 100000;",
       [TIMING + "test_latency_per_hop"], "every rep lasts 100 us longer than it did"),
    # ---- pingpong_kernels.cu ----
    _m("pingpong_digest_of_the_ping", "pingpong_kernels.cu", "initiate",
       "digest ^= v;", "digest ^= v - 1;", [RR + "test_pingpong_digest_over_an_odd_number_of_trips"],
       "the digest xors the ping rather than its echo"),
    _m("pingpong_warmup_digest_dropped", "pingpong_kernels.cu", "initiate",
       "o[rep].digest = digest;", "o[rep].digest = rep == 0 ? 0ull : digest;",
       [RR + "test_pingpong_digest_over_an_odd_number_of_trips"],
       "the warm-up rep's digest is left out"),
    _m("pingpong_rep_time_plus_100us", "pingpong_kernels.cu", "initiate",
       "o[rep].ns = t1 - t0;", "o[rep].ns = t1 - t0 + 100000;", [RR + "test_short_pingpong_reps_are_not_padded"],
       "every rep lasts 100 us longer than it did"),
    # ---- atomics_kernels.cu ----
    _m("atomics_chain_digest_adds", "atomics_kernels.cu", "atomics_chain_kernel",
       "digest ^= x;", "digest += x;", [AT + "test_every_cell_clean"],
       "the chain's digest is a sum of the returns"),
    _m("atomics_contended_digest_sums", "atomics_kernels.cu", "atomics_contended_kernel",
       "digest = warp_xor(digest);", "digest = warp_sum(digest);",
       [RR + "test_atomics_digest_over_an_odd_number_of_ops"],
       "the contended digest sums the lanes' digests"),
    _m("atomics_chain_rep_time_plus_100us", "atomics_kernels.cu", "atomics_chain_kernel",
       "o[r].ns = t1 - t0;", "o[r].ns = t1 - t0 + 100000;", [TIMING + "test_atomics_per_op"],
       "every rep of a chain lasts 100 us longer than it did"),
    # ---- bwcurve_kernels.cu ----
    _m("bwcurve_warmup_sum_off", "bwcurve_kernels.cu", "bwcurve_kernel",
       "Sum a{0ull, 0ull, 0ull};", "Sum a{r == 0 ? 1ull : 0ull, 0ull, 0ull};",
       [BW + "test_loopback_every_size_clean"], "the warm-up rep's S is off by one per warp"),
    _m("bwcurve_first_timed_rep_sum_off", "bwcurve_kernels.cu", "bwcurve_kernel",
       "Sum a{0ull, 0ull, 0ull};", "Sum a{0ull, r == 1 ? 1ull : 0ull, 0ull};",
       [BW + "test_loopback_every_size_clean"], "timed rep 1's S is off by one per warp"),
    _m("bwcurve_rep_end_late", "bwcurve_kernels.cu", "bwcurve_kernel",
       "atomicMax(&acc->t_end, (unsigned long long)gtimer());",
       "atomicMax(&acc->t_end, (unsigned long long)gtimer() + 100000);",
       [RR + "test_short_bwcurve_reps_are_not_padded"], "every rep's end stamp is 100 us late"),
    # ---- alltoall_kernels.cu ----
    _m("a2a_check_fold_by_unit", "alltoall_kernels.cu", "a2a_check",
       "fold6(u / (kGranuleBytes / kUnitBytes))", "fold6(u)",
       [A2A + "test_single_rank_every_size_clean", A2A + "test_same_device_every_cell_clean"],
       "the received blocks' X is folded per unit, not per granule; the word check still passes"),
    _m("a2a_first_bad_odd_word_late", "alltoall_kernels.cu", "a2a_check",
       "first = min(first, 8 * k0 + 8);", "first = min(first, 8 * k0 + 16);",
       [A2A + "test_an_armed_fault_fails_exactly_its_cell_and_size", EDGES + "test_grids_and_faults_at_the_edges"],
       "a bad odd word is reported one word late"),
    _m("a2a_salt_sender_receiver_swapped", "alltoall_kernels.cu", "place",
       "write_salt(P->seed, P->rank, P->to[b], seq)", "write_salt(P->seed, P->to[b], P->rank, seq)",
       [A2A + "test_same_device_every_cell_clean"],
       "a sender stores the pattern of the reverse pair; identical on the diagonal"),
    # ---- allreduce_kernels.cu ----
    _m("oneshot_fault_halves_swapped", "allreduce_kernels.cu", "ar_store",
       "if (fb & 8u) acc[2 * i + 1] += 1ull;\n      else acc[2 * i] += 1ull;",
       "if (fb & 8u) acc[2 * i] += 1ull;\n      else acc[2 * i + 1] += 1ull;",
       [AR + "test_an_armed_fault_fails_exactly_one_row_and_size", EDGES + "test_grids_and_faults_at_the_edges"],
       "the armed fault adds to the other word of its vector"),
    _m("oneshot_fault_every_timed_rep", "allreduce_kernels.cu", "allreduce_kernel",
       "(r == 1u && k == P.fault_k)", "(r >= 1u && k == P.fault_k)",
       [AR + "test_an_armed_fault_fails_exactly_one_row_and_size", EDGES + "test_grids_and_faults_at_the_edges"],
       "the armed fault acts in every timed rep"),
    _m("oneshot_full_unit_words_swapped", "allreduce_kernels.cu", "ar_store",
       "stg_pair(base + ar_vec_off<kLaneBytes>(c.lane, i), acc[2 * i], acc[2 * i + 1]);\n  } else {",
       "stg_pair(base + ar_vec_off<kLaneBytes>(c.lane, i), acc[2 * i + 1], acc[2 * i]);\n  } else {",
       [AR + "test_single_rank_every_size_clean"], "a whole unit leaves with the words of each vector swapped"),
    # ---- allreduce_twoshot_kernels.cu ----
    _m("twoshot_drop_mode_ignored", "allreduce_twoshot_kernels.cu", "put",
       "put_ranks<kLaneBytes, true>", "put_ranks<kLaneBytes, false>",
       [AR2 + "test_a_dropped_unit_reads_as_zeros_because_every_rep_clears_the_output"],
       "a dropped unit is stored, with the fault's flipped word"),
    _m("twoshot_fault_every_timed_rep", "allreduce_twoshot_kernels.cu", "allreduce_twoshot_kernel",
       "(r == 1u && k == P.fault_k)", "(r >= 1u && k == P.fault_k)",
       [RR + "test_twoshot_fault_acts_in_timed_rep_1_of_3_only"], "the armed fault acts in every timed rep"),
    _m("twoshot_fault_on_neighbour_word", "allreduce_twoshot_kernels.cu", "allreduce_twoshot_kernel",
       "? P.fault_word : ~0ull", "? P.fault_word ^ 1ull : ~0ull",
       [AR2 + "test_grids_and_faults_at_the_edges"], "the armed fault lands on the other word of its vector"),
    # ---- allreduce_ll_kernels.cu ----
    _m("ll_last_word_off", "allreduce_ll_kernels.cu", "ll_rep",
       "const uint64_t v = acc - salts;", "const uint64_t v = acc - salts + (w == 1 ? 1ull : 0ull);",
       [LL + "test_tiny_ladders_and_the_ladder_cut_at_1_mib"],
       "word 1 of every size is one too large"),
    _m("ll_x_folded_per_line", "allreduce_ll_kernels.cu", "ll_rep",
       "fold6((uint32_t)(i / (kGranuleWords / 32)))", "fold6((uint32_t)i)",
       [LL + "test_tiny_ladders_and_the_ladder_cut_at_1_mib"],
       "the output's X is folded per line, not per granule; the word check still passes"),
    _m("ll_fault_to_every_other_peer", "allreduce_ll_kernels.cu", "ll_rep",
       "(w == fw && t == P.fault_dst)", "(w == fw && t != P.fault_dst)",
       [LL + "test_a_corrupted_packet_fails_only_its_receiver_and_size"],
       "the corrupted packet goes to every receiver but the armed one"),
    # ---- allreduce_ring_kernels.cu ----
    _m("ring_own_store_words_swapped", "allreduce_ring_kernels.cu", "ring_unit",
       "if (st.own) stg_pair(P.out + base + off, w0, w1);", "if (st.own) stg_pair(P.out + base + off, w1, w0);",
       [RING + "test_single_rank_every_size_clean"],
       "a rank's own chunk lands with the words of each vector swapped; its pushes are right"),
    _m("ring_fault_in_the_other_phase", "allreduce_ring_kernels.cu", "ring_rep",
       "st.phase == P.fault_phase ? fw : ~0ull", "st.phase != P.fault_phase ? fw : ~0ull",
       [RING + "test_a_faulted_push_fails_exactly_the_rows_the_restatement_names"],
       "the armed push fault acts in the other phase"),
    _m("ring_fault_halves_swapped", "allreduce_ring_kernels.cu", "ring_unit",
       "if (hit & 8u) w1 ^= 1ull;\n      else w0 ^= 1ull;", "if (hit & 8u) w0 ^= 1ull;\n      else w1 ^= 1ull;",
       [RING + "test_a_faulted_push_fails_exactly_the_rows_the_restatement_names"],
       "the armed push fault flips the other word of its vector"),
    # ---- allreduce_push_kernels.cu ----
    _m("push_ldst_fault_halves_swapped", "allreduce_push_kernels.cu", "reduce_ldst",
       "if (fb & 8u) w1 += 1ull;\n          else w0 += 1ull;", "if (fb & 8u) w0 += 1ull;\n          else w1 += 1ull;",
       [PUSH + "test_each_fault_fails_exactly_the_rows_and_words_the_restatement_names"],
       "the ld/st reduce-scatter's fault adds to the other word of its vector"),
    _m("push_mode_2_disarmed", "allreduce_push_kernels.cu", "allreduce_push_kernel",
       "armed && P.fault_mode < 3u ?", "armed && P.fault_mode < 2u ?",
       [PUSH + "test_each_fault_fails_exactly_the_rows_and_words_the_restatement_names"],
       "the doubled reduction (mode 2) never happens"),
    _m("push_gather_fault_one_word_late", "allreduce_push_kernels.cu", "allreduce_push_kernel",
       "P.fault_mode == 3u ? P.fault_word : ~0ull", "P.fault_mode == 3u ? P.fault_word + 1 : ~0ull",
       [PUSH + "test_each_fault_fails_exactly_the_rows_and_words_the_restatement_names"],
       "the all-gather's fault (mode 3) flips the word after the armed one"),
    # ---- allreduce_nvls_kernels.cu ----
    _m("nvls_vector_words_swapped", "allreduce_nvls_kernels.cu", "reduce_store",
       "uint64_t w0 = w[2 * i], w1 = w[2 * i + 1];", "uint64_t w0 = w[2 * i + 1], w1 = w[2 * i];",
       [NVLS + "test_clean_ladders_on_every_grid"], "every multicast store swaps the two words of its vector"),
    _m("nvls_fault_on_every_other_vector", "allreduce_nvls_kernels.cu", "reduce_store",
       "if (hit && off == (fb & ~15u))", "if (hit && off != (fb & ~15u))",
       [NVLS + "test_each_fault_fails_exactly_the_words_the_restatement_names"],
       "the armed fault flips a word of every vector of its unit but the armed one"),
    _m("nvls_fault_in_the_warmup", "allreduce_nvls_kernels.cu", "allreduce_nvls_kernel",
       "(r == 1u && k == P.fault_k)", "(r == 0u && k == P.fault_k)",
       [NVLS + "test_each_fault_fails_exactly_the_words_the_restatement_names"],
       "the armed fault acts in the warm-up rep instead of timed rep 1"),
    # ---- allreduce_path.cuh ----
    _m("ar_add_low_carry_lost", "allreduce_path.cuh", "ar_add",
       "acc[2 * i] += pack64(v.x, v.y);",
       "acc[2 * i] = (((acc[2 * i] >> 32) + v.y) << 32) | (uint32_t)((uint32_t)acc[2 * i] + v.x);",
       [AR + "test_same_device_every_row_clean"],
       "the even word's 64-bit add loses the carry out of its low half"),
    _m("ar_check_clear_stores_the_word_back", "allreduce_path.cuh", "ar_check_clear",
       "stg_v4(p + v, make_uint4(0u, 0u, 0u, 0u));", "stg_v4(p + v, q);",
       [AR + "test_a_dropped_unit_is_seen_whatever_the_output_held_before",
        AR2 + "test_a_dropped_unit_reads_as_zeros_because_every_rep_clears_the_output"],
       "the check leaves the word it read instead of 0, so a unit a later rep drops still reads right"),
    _m("ar_check_clear_first_one_word_late", "allreduce_path.cuh", "ar_check_clear",
       "first = min(first, 8 * k0);", "first = min(first, 8 * k0 + 8);",
       [AR + "test_an_armed_fault_fails_exactly_one_row_and_size", EDGES + "test_grids_and_faults_at_the_edges"],
       "a bad even word is reported one word late"),
    _m("ar_check_stores_the_sum_back", "allreduce_path.cuh", "ar_check",
       "out[w] = 0ull;", "out[w] = allreduce_word(P.seed, P.n, w);",
       [LL + "test_an_unstored_word_is_seen_whatever_the_output_held_before"],
       "the LL check leaves the right sum instead of 0, so a word the next size does not store still reads right"),
    _m("put_ranks_fault_to_the_next_rank", "allreduce_path.cuh", "put_ranks",
       "== u ? P.fault_dst : ~0u", "== u ? P.fault_dst + 1 : ~0u",
       [AR2 + "test_grids_and_faults_at_the_edges"],
       "the two-shot's and the push's armed store fault acts on the next rank's copy"),
    # ---- timed_rep.cuh ----
    _m("closing_timer_read_100us_late", "timed_rep.cuh", "globaltimer_after",
       "return t;", "return t + 100000;",
       [TIMING + "test_latency_per_hop", TIMING + "test_pingpong_per_trip"],
       "every rep of latency and pingpong lasts 100 us longer (atomics open with this read too, so theirs do not)"),
    _m("closing_timer_read_before_the_opening", "timed_rep.cuh", "globaltimer_after",
       "return t;", "return t - 100000;",
       [TIMING + "test_latency_per_hop", TIMING + "test_pingpong_per_trip"],
       "every closing read is 100 us early, before its opening read where that is a plain read (latency, pingpong)"),
    # ---- measure.cc ----
    _m("fold_checks_last_rep_only", "measure.cc", "fold_checks",
       "out->bad_words[idx][k] += g.diag[0];", "out->bad_words[idx][k] = g.diag[0];",
       [MC + "test_an_armed_fault_fails_exactly_its_cell_and_size"],
       "a size's bad_words is its last rep's, not the sum over its reps"),
    _m("fold_checks_first_one_word_late", "measure.cc", "fold_checks",
       "first = std::min(first, (uint64_t)~g.diag[2]);", "first = std::min(first, (uint64_t)~g.diag[2] + 8);",
       [MC + "test_an_armed_fault_fails_exactly_its_cell_and_size"], "first_bad names the word after"),
    _m("summarize_warmup_digest_dropped", "measure.cc", "summarize",
       "digest ^= rep[k].digest;", "if (k > 0) digest ^= rep[k].digest;",
       [LAT + "test_loopback_chase_digest_and_times", PP + "test_every_cell_clean"],
       "the cell's digest leaves out the warm-up rep"),
    _m("ladder_t0_from_the_minimum", "measure.cc", "ladder_times",
       "out->t0_ns[idx] = out->ns_median[idx][0];", "out->t0_ns[idx] = out->ns_min[idx][0];",
       [LADDER_TIMING + "test_windows_fit_in_the_call"], "t0_ns is the smallest size's minimum, not its median"),
    _m("word_checks_first_one_word_late", "measure.cc", "word_checks",
       "? ~first_bad_n[k] : UINT64_MAX", "? ~first_bad_n[k] + 8 : UINT64_MAX",
       [AR + "test_an_armed_fault_fails_exactly_one_row_and_size"],
       "the all-reduces' and the all-to-all's first_bad names the word after"),
]

# The translation units of libcdprobe.so that compile each source file (a .cu or .cc is its own unit).
HEADER_UNITS = {
    "datapath.cuh": ["probe_kernels.cu", "bwcurve_kernels.cu", "alltoall_kernels.cu", "allreduce_kernels.cu",
                     "allreduce_twoshot_kernels.cu", "allreduce_ll_kernels.cu", "allreduce_ring_kernels.cu",
                     "allreduce_push_kernels.cu", "allreduce_nvls_kernels.cu"],
    "allreduce_path.cuh": ["allreduce_kernels.cu", "allreduce_twoshot_kernels.cu", "allreduce_ll_kernels.cu",
                           "allreduce_ring_kernels.cu", "allreduce_push_kernels.cu", "allreduce_nvls_kernels.cu"],
    "timed_rep.cuh": ["latency_kernels.cu", "pingpong_kernels.cu", "atomics_kernels.cu", "measure.cc"],
}


def units(m):
    """The translation units a change to m's file recompiles."""
    return HEADER_UNITS.get(m["file"], [m["file"]])


def by_name(name):
    found = [m for m in MUTANTS if m["name"] == name]
    assert len(found) == 1, (name, len(found))
    return found[0]
