// plan.cc — see plan.h.  Pure integer host code; exported through the C ABI as
// cdprobe_plan() so it can be checked without a GPU.
#include "plan.h"

#include <string.h>

namespace cdp {

int partner_of(uint32_t n, uint32_t r, uint32_t i) {
  if (n < 2 || i >= n) return -1;
  const uint32_t ne = (n & 1u) ? n + 1 : n;  // pad odd n with a dummy rank
  const uint32_t m = ne - 1;                 // odd modulus
  if (r >= m) return -1;
  uint32_t p;
  if (i == ne - 1) {
    // the fixed rank meets the x with 2x == r (mod m); 2^-1 mod m = (m + 1) / 2
    p = (uint32_t)(((uint64_t)r * ((m + 1) / 2)) % m);
  } else {
    const uint32_t j = (r + m - (i % m)) % m;
    p = (j == i) ? ne - 1 : j;
  }
  return p < n ? (int)p : -1;
}

static uint64_t round_up(uint64_t v, uint64_t a) { return (v + a - 1) / a * a; }

int make_plan(uint32_t n, uint64_t bytes, uint32_t mode, uint32_t flags, Plan* out) {
  if (n < 1 || n > (uint32_t)kMaxRanks || out == nullptr) return CDPROBE_ERR_ARG;
  Plan p;
  memset(p.partner, -1, sizeof(p.partner));
  p.n = n;
  const uint32_t peers = n - 1;
  p.diag = (n == 1) || (flags & CDPROBE_FLAG_LOCAL_DIAG);
  p.full = (mode == CDPROBE_MODE_FULL);
  switch (mode) {
    case CDPROBE_MODE_REACH_ONLY:
      p.bpp = 64ull << 10;
      break;
    case CDPROBE_MODE_SLICED:
      p.bpp = bytes / (peers ? peers : 1) / 128 * 128;
      break;
    case CDPROBE_MODE_FULL:
      p.bpp = bytes / 128 * 128;
      break;
    default:
      return CDPROBE_ERR_ARG;
  }
  if (p.bpp < 128 || p.bpp > (16ull << 30)) return CDPROBE_ERR_ARG;
  p.n_slots = peers + (p.diag ? 1u : 0u);
  p.diag_slot = peers;
  p.n_slices = p.full ? 1u : p.n_slots;
  p.src_bytes = (uint64_t)p.n_slices * p.bpp;
  p.land_bytes = (uint64_t)p.n_slots * p.bpp;
  p.src_off = kCtrlBytes;
  p.land_off = p.src_off + round_up(p.src_bytes, kVmmGranule);
  p.alloc_bytes = p.land_off + round_up(p.land_bytes, kVmmGranule);
  p.rounds = n == 1 ? 0u : ((n & 1u) ? n : n - 1);
  for (uint32_t r = 0; r < p.rounds; ++r)
    for (uint32_t i = 0; i < n; ++i) p.partner[r][i] = (int8_t)partner_of(n, r, i);
  *out = p;
  return CDPROBE_OK;
}

MemcpyCell memcpy_cell(const Plan& pl, uint32_t op, uint32_t g, uint32_t j) {
  // a pull moves the slice g reads from j to g; a push moves the slice j reads from g to j
  const bool push = op == CDPROBE_OP_WRITE;
  const uint32_t reader = push ? j : g, owner = push ? g : j;
  MemcpyCell c;
  c.src_rank = owner;
  c.src_off = cell_offset(pl, CDPROBE_OP_READ, reader, owner);
  c.first_word = (uint64_t)cell_slice(pl, reader, owner) * (pl.bpp / 8);
  c.dst_rank = reader;
  c.dst_off = (uint64_t)owner * pl.bpp;
  return c;
}

uint32_t ce_a2a_queues(uint32_t n, bool diag, uint32_t n_local, const int* ordinal, int* worst) {
  const uint32_t per_rank = 1u + (n - 1u) + (diag ? 1u : 0u);
  uint32_t most = 0;
  *worst = n_local ? ordinal[0] : -1;
  for (uint32_t li = 0; li < n_local; ++li) {
    uint32_t here = 0;
    for (uint32_t lj = 0; lj < n_local; ++lj) here += ordinal[lj] == ordinal[li] ? per_rank : 0u;
    if (here > most || (here == most && ordinal[li] < *worst)) {
      most = here;
      *worst = ordinal[li];
    }
  }
  return most;
}

}  // namespace cdp

extern "C" int cdprobe_plan(uint32_t n, uint64_t bytes, uint32_t mode, uint32_t flags, cdprobe_plan_t* out) {
  if (out == nullptr) return CDPROBE_ERR_ARG;
  cdp::Plan p;
  const int rc = cdp::make_plan(n, bytes, mode, flags, &p);
  if (rc != CDPROBE_OK) return rc;
  memset(out, 0, sizeof(*out));
  out->abi = CDPROBE_ABI_VERSION;
  out->n = p.n;
  out->rounds = p.rounds;
  out->n_slots = p.n_slots;
  out->n_slices = p.n_slices;
  out->bytes_per_pair = p.bpp;
  out->src_bytes = p.src_bytes;
  out->land_bytes = p.land_bytes;
  memset(out->partner, -1, sizeof(out->partner));
  for (uint32_t r = 0; r < p.rounds; ++r)
    for (uint32_t i = 0; i < p.n; ++i) out->partner[r][i] = p.partner[r][i];
  return CDPROBE_OK;
}
