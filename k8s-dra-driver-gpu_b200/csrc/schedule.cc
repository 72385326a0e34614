// schedule.cc — the phase table one rank's persistent kernel walks (host only, pure function).
//
// SURVEY.md §8(d)/(e): rounds of the tournament x {write, read}, verification of what peers
// stored, the link wake-up phase.  Every rank must produce the same NUMBER of phases with the
// same barrier kinds (the device barrier is indexed by phase), whatever its own role in a phase.
// Exported through the C ABI as cdprobe_schedule() so the invariants are tested without a GPU
// (tests/test_schedule.py).
#include "schedule.h"

#include <string.h>

namespace cdp {

// Phase table of local rank li (SURVEY.md §8d schedule: rounds x {read, write}, then verify).
// With CDPROBE_FLAG_OVERLAP_VERIFY the landing slot a partner filled in round r is verified by
// the last `verify_ctas` CTAs while the other CTAs drive round r + 1 over NVLink: local HBM has
// ~8x the bandwidth of the link, so the verify disappears from the critical path.
int make_phases(const ScheduleInput& in, Phase* phases, uint32_t* n_phases, uint32_t* peer_mask) {
  const Plan& pl = *in.plan;
  const uint32_t g = in.rank;
  const uint32_t ops = in.ops;
  const uint32_t ctas = in.ctas;
  auto pair_ok = [&](uint32_t a, uint32_t b) {
    return in.status == nullptr || (in.status[a][b] == 0 && in.status[b][a] == 0);
  };
  uint32_t n = 0;
  auto set_job = [&](Job& j, uint8_t kind, int peer, uint32_t slot, uint32_t writer, uint32_t cta0, uint32_t nctas) {
    memset(&j, 0, sizeof(j));
    j.kind = kind;
    j.peer = (int8_t)peer;
    j.slot = (uint8_t)slot;
    j.writer = (uint8_t)writer;
    j.cta0 = (uint16_t)cta0;
    j.nctas = (uint16_t)nctas;
  };
  bool overflow = false;
  Phase scratch;
  int cur_round = -1;               // tournament round of the phases being pushed (-1: local-only phases)
  int phase_round[kMaxPhases];      // per phase: the round whose pairing decides which NVLink ports it loads
  bool is_write_phase[kMaxPhases] = {}, is_read_phase[kMaxPhases] = {};  // the W / R phase of a tournament round
  auto push = [&](uint8_t kind, int peer, uint32_t slot, uint32_t writer) -> Phase& {
    if (n >= (uint32_t)kMaxPhases) {
      overflow = true;
      return scratch;
    }
    phase_round[n] = cur_round;
    Phase& p = phases[n++];
    memset(&p, 0, sizeof(p));
    set_job(p.job[0], kind, peer, slot, writer, 0, ctas);
    return p;
  };
  // Overlapped verify is a property of the DOMAIN's schedule (every rank must walk the same number of phases),
  // so it may not depend on this rank's CTA count — a rank throttled to 2 CTAs next to 148-CTA peers once
  // fell back to serial verify on its own, grew extra phases and dead-locked the barrier sequence.  Only the
  // split adapts: verify_ctas when there is room, half the CTAs on a small grid, and on a single CTA both
  // jobs cover CTA 0 (the kernel runs a CTA's jobs one after the other).
  const bool overlap = (in.flags & CDPROBE_FLAG_OVERLAP_VERIFY) && (ops & CDPROBE_OP_WRITE) && pl.rounds > 0 &&
                       in.verify_ctas > 0;
  const uint32_t vctas = ctas >= 2 * in.verify_ctas ? in.verify_ctas : (ctas >= 2 ? ctas / 2 : ctas);
  const uint32_t link_ctas = ctas >= 2 ? ctas - vctas : ctas;  // CTAs of the NVLink job when a verify rides along
  struct Pending {
    bool have = false, ok = false;
    uint32_t slot = 0, writer = 0;
    uint32_t wphase = 0;  // phase in which the writer stores into the slot
  } pend;
  uint32_t write_phase_into[kMaxRanks] = {};  // [landing slot] -> phase in which its remote writer stores (serial verify)
  auto attach = [&](Phase& p) {  // give the tail CTAs of phase p the pending verify
    if (!pend.have) return;
    if (p.job[0].kind != kJobNone) p.job[0].nctas = (uint16_t)link_ctas;
    set_job(p.job[1], pend.ok ? kJobVerify : kJobNone, (int)g, pend.slot, pend.writer, ctas >= 2 ? link_ctas : 0, vctas);
    if (pend.ok && pend.writer != g) p.job[1].salt = pend.wphase + 1;  // barrier that closes the writer's phase
    pend.have = false;
  };
  // Bidirectional (default): both ranks of a pair issue at once, so every NVLink port carries
  // data in both directions.  CDPROBE_FLAG_UNIDIRECTIONAL splits a round in two halves — the
  // lower rank of the pair issues first, then the higher — so each ordered pair is measured
  // with its two ports carrying payload one way only (the classic per-link figure).
  const bool uni = (in.flags & CDPROBE_FLAG_UNIDIRECTIONAL) != 0;
  if (pl.rounds > 0) {
    // Phase 0: link wake-up.  After a stretch of idleness the first NVLink transfer can pay a fixed
    // start-up cost before data flows, which would make the first timed phase of a cold probe report a
    // fraction of the link's rate and fail healthy pairs.  Every rank
    // streams a small prefix of its round-0 partner's slice, untimed; the phase always exists (all
    // ranks need the same barrier sequence) and each rank decides its own byte count at launch (0 when
    // its previous run ended less than warm_idle_ms ago).
    cur_round = 0;
    const int p0 = pl.partner[0][g];
    const bool ok0 = p0 >= 0 && pair_ok(g, (uint32_t)p0);
    push(ok0 ? kJobWarm : kJobNone, ok0 ? p0 : (int)g, ok0 ? slot_of(g, (uint32_t)p0) : 0, 0);
  }
  for (uint32_t r = 0; r < pl.rounds; ++r) {
    cur_round = (int)r;
    const int p = pl.partner[r][g];
    const bool ok = p >= 0 && pair_ok(g, (uint32_t)p);
    const uint32_t slot = ok ? slot_of(g, (uint32_t)p) : 0;
    for (int half = 0; half < (uni ? 2 : 1); ++half) {
      const bool i_active = !uni || ((half == 0) == ((int)g < p));
      const bool p_active = !uni || !i_active;
      const bool mine = ok && i_active;
      // write first, then read: the slot the partner fills during the write phase is verified by the
      // spare CTAs during the read phase of the SAME round, so no verify is left over at the end
      if (ops & CDPROBE_OP_WRITE) {
        Phase& ph = push(mine ? kJobWrite : kJobNone, mine ? p : (int)g, slot, 0);
        if (p >= 0 && p_active) write_phase_into[slot_of((uint32_t)p, g)] = n - 1;
        if (!overflow) is_write_phase[n - 1] = true;
        if (overlap) {
          attach(ph);
          if (p >= 0 && p_active) {  // what the partner stores into my landing area during this phase
            pend.have = true;
            pend.ok = ok;
            pend.slot = slot_of((uint32_t)p, g);
            pend.writer = (uint32_t)p;
            pend.wphase = n - 1;
          }
        }
      }
      if (ops & CDPROBE_OP_READ) {
        Phase& ph = push(mine ? kJobRead : kJobNone, mine ? p : (int)g, slot, 0);
        if (!overflow) is_read_phase[n - 1] = true;
        if (overlap) attach(ph);
      }
    }
  }
  // Loop-back (N = 1, or CDPROBE_FLAG_LOCAL_DIAG): same shape as a round — write the diagonal slot,
  // then read the source slice on half the CTAs while the other half verifies what was just written
  // (both jobs are HBM-bound, hence the near-even split).  One barrier fewer than read / write / verify.
  cur_round = -1;
  const bool diag_overlap = pl.diag && (in.flags & CDPROBE_FLAG_OVERLAP_VERIFY) && (ops & CDPROBE_OP_WRITE) &&
                            (ops & CDPROBE_OP_READ);  // not a function of ctas: see `overlap` above
  if (pl.diag) {
    if (ops & CDPROBE_OP_WRITE) push(kJobWrite, (int)g, pl.diag_slot, 0);
    if (ops & CDPROBE_OP_READ) {
      Phase& ph = push(kJobRead, (int)g, pl.diag_slot, 0);
      if (diag_overlap) {
        // measured at N = 1 with an even split: the verify half (reading lines that were just written)
        // runs ~5 % slower than the source read, so it gets 33/64 of the CTAs (76 of 148)
        if (ctas >= 2) {
          uint32_t half = (ctas * 33u + 32u) / 64u;
          if (half < 1) half = 1;
          if (half >= ctas) half = ctas - 1;
          ph.job[0].nctas = (uint16_t)(ctas - half);
          set_job(ph.job[1], kJobVerify, (int)g, pl.diag_slot, g, ctas - half, half);
        } else {
          set_job(ph.job[1], kJobVerify, (int)g, pl.diag_slot, g, 0, 1);  // one CTA: read, then verify
        }
      }
    }
  }
  if (ops & CDPROBE_OP_WRITE) {
    if (overlap) {
      // With reads in the schedule every write phase is followed by a read phase that carried its
      // verify, on every rank.  Write-only probes keep one trailing verify phase — always present (a
      // rank that sat out the last round of an odd-sized domain pushes an idle phase) so that every
      // rank has the same number of barriers.
      if (!(ops & CDPROBE_OP_READ)) {
        Phase& ph = push(pend.have && pend.ok ? kJobVerify : kJobNone, (int)g, pend.slot, pend.writer);
        if (ph.job[0].kind == kJobVerify && pend.writer != g) ph.job[0].salt = pend.wphase + 1;
      }
      pend.have = false;
      if (pl.diag && !diag_overlap) push(kJobVerify, (int)g, pl.diag_slot, g);
    } else {
      for (uint32_t s = 0; s < pl.n_slots; ++s) {
        uint32_t writer;
        bool ok;
        if (pl.diag && s == pl.diag_slot) {
          if (diag_overlap) continue;  // already verified next to the loop-back read
          writer = g;
          ok = true;
        } else {
          writer = s < g ? s : s + 1;
          ok = pair_ok(g, writer);
        }
        Phase& ph = push(ok ? kJobVerify : kJobNone, (int)g, s, writer);
        if (ok && writer != g) ph.job[0].salt = write_phase_into[s] + 1;
      }
    }
  }
  if (overflow) {
    *n_phases = 0;
    return CDPROBE_ERR_ARG;
  }
  // ---- closing barrier of every phase: who must this rank exchange flags with? -------------------
  // The barrier between phase p and p + 1 has to order (a) the data dependencies — the verify that
  // follows a write, the publication of write checksums — and (b) the exclusivity of NVLink ports the
  // per-pair GB/s relies on: nobody may start loading a port that a transfer of the previous phase is
  // still using.  With A(x, p) = the partner of rank x in phase p, the ranks whose phase-p or
  // phase-(p+1) traffic shares a port with this rank's are
  //     M = { A(g,p), A(g,p+1), A(A(g,p+1), p), A(A(g,p), p+1) }
  // (symmetric: y in M(g) <=> g in M(y), so every rank waited for also signals).  An all-rank exchange
  // (round 1: 15 of them at N = 8, 6-10 us each) is kept at the open and at the close of a run, and
  // everywhere with CDPROBE_FLAG_ALL_RANK_BARRIERS.
  const uint32_t everyone = (pl.n >= 32 ? 0xffffffffu : ((1u << pl.n) - 1u)) & ~(1u << g);
  auto partner_in = [&](int round, int x) -> int {
    return (round >= 0 && x >= 0) ? (int)pl.partner[round][x] : -1;
  };
  for (uint32_t p = 0; p < n; ++p) {
    uint32_t m = 0;
    if (p + 1 == n) {
      m = everyone;  // verdicts must be visible before the rows are written
    } else if ((in.flags & CDPROBE_FLAG_ALL_RANK_BARRIERS) && (phase_round[p] >= 0 || phase_round[p + 1] >= 0)) {
      m = everyone;
    } else {
      const int r0 = phase_round[p], r1 = phase_round[p + 1];
      const int a = partner_in(r0, (int)g), b = partner_in(r1, (int)g);
      const int cand[4] = {a, b, partner_in(r0, b), partner_in(r1, a)};
      for (int c : cand)
        if (c >= 0 && (uint32_t)c != g) m |= 1u << c;
      // Write -> read of the same pair (bidirectional schedule): the read does not need the partner's ports to be
      // quiet — they are the pair's own — only the verify that rides along needs the partner's data, and that job
      // waits for the partner's signal itself.  So nobody waits at this barrier: the rank releases its own CTAs and
      // then signals the partner (post_mask).  ~3 us less per round on the critical path (r02_trace_n8).
      const bool uni_mode = (in.flags & CDPROBE_FLAG_UNIDIRECTIONAL) != 0;
      if (!uni_mode && !(in.flags & CDPROBE_FLAG_PAIR_BARRIERS) && r0 >= 0 && r0 == r1 && is_write_phase[p] && is_read_phase[p + 1]) {
        phases[p].post_mask = m;
        m = 0;
      }
    }
    phases[p].sync_mask = m;
  }
  *n_phases = n;
  uint32_t mask = 0;
  for (uint32_t j = 0; j < pl.n; ++j)
    if (j != g && pair_ok(g, j)) mask |= 1u << j;
  *peer_mask = mask;
  return CDPROBE_OK;
}


}  // namespace cdp

extern "C" int cdprobe_schedule(uint32_t n, uint32_t rank, uint64_t bytes, uint32_t mode, uint32_t ops, uint32_t flags,
                                uint32_t ctas, uint32_t verify_ctas, cdprobe_schedule_t* out) {
  if (out == nullptr || rank >= n || ctas == 0 || ctas > 65535u) return CDPROBE_ERR_ARG;
  cdp::Plan pl;
  int rc = cdp::make_plan(n, bytes, mode, flags, &pl);
  if (rc != CDPROBE_OK) return rc;
  if (ops == 0) ops = CDPROBE_OP_READ | CDPROBE_OP_WRITE;
  if (!(flags & CDPROBE_FLAG_SERIAL_VERIFY)) flags |= CDPROBE_FLAG_OVERLAP_VERIFY;
  cdp::ScheduleInput in;
  in.plan = &pl;
  in.rank = rank;
  in.ops = ops;
  in.flags = flags;
  in.ctas = ctas;
  in.verify_ctas = verify_ctas ? verify_ctas : 32u;
  in.status = nullptr;
  cdp::Phase ph[cdp::kMaxPhases];
  uint32_t np = 0, mask = 0;
  rc = cdp::make_phases(in, ph, &np, &mask);
  memset(out, 0, sizeof(*out));
  out->abi = CDPROBE_ABI_VERSION;
  if (rc != CDPROBE_OK) return rc;
  out->n_phases = np;
  out->peer_mask = mask;
  for (uint32_t p = 0; p < np; ++p) {
    for (int jb = 0; jb < 2; ++jb) {
      const cdp::Job& j = ph[p].job[jb];
      out->kind[jb][p] = j.kind;
      out->peer[jb][p] = j.peer;
      out->slot[jb][p] = j.slot;
      out->writer[jb][p] = j.writer;
      out->cta0[jb][p] = j.cta0;
      out->nctas[jb][p] = j.nctas;
    }
    out->sync_mask[p] = (uint16_t)(ph[p].sync_mask & mask);
    out->post_mask[p] = (uint16_t)(ph[p].post_mask & mask);
    out->wait_barrier[0][p] = (uint8_t)(ph[p].job[0].kind == cdp::kJobVerify ? ph[p].job[0].salt : 0);
    out->wait_barrier[1][p] = (uint8_t)(ph[p].job[1].kind == cdp::kJobVerify ? ph[p].job[1].salt : 0);
    out->sync_all[p] = (uint8_t)(mask != 0 && (ph[p].sync_mask & mask) == mask);
  }
  return CDPROBE_OK;
}
