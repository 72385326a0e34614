// plan.h — tournament schedule and slice arithmetic of a probe (host only).
//
// SURVEY.md §8(d)/(e): ordered pairs (i, j), i != j, are partitioned by issuer
// i; round r pairs i with partner(i, r) (circle method) so every GPU has
// exactly one partner per round and owns both endpoints of the pair.
#pragma once
#include <stdint.h>

#include "../../include/cdprobe.h"
#include "probe_types.h"

namespace cdp {

struct Plan {
  uint32_t n = 0;          // ranks
  uint32_t rounds = 0;     // tournament rounds
  uint32_t n_slots = 0;    // landing slots per rank
  uint32_t n_slices = 0;   // source slices per rank
  uint32_t diag_slot = 0;  // slot/slice used by the loop-back (valid when diag)
  bool diag = false;
  bool full = false;
  uint64_t bpp = 0;        // bytes per pair
  uint64_t src_bytes = 0, land_bytes = 0;
  uint64_t src_off = 0, land_off = 0, alloc_bytes = 0;
  int8_t partner[kMaxRanks][kMaxRanks];  // [round][rank]
};

// Partner of rank i in round r of an n-rank tournament, -1 when i sits out (odd n).
int partner_of(uint32_t n, uint32_t r, uint32_t i);
// Slot of issuer i inside owner j's buffers (its index among j's peers).
inline uint32_t slot_of(uint32_t i, uint32_t j) { return i < j ? i : i - 1; }
// Where cell (issuer i, target j) lives in j's allocation: the landing slot i writes and the source slice i reads
// (in full mode every reader reads slice 0).  The loop-back cell i == j uses the diagonal slot.
inline uint32_t cell_slot(const Plan& pl, uint32_t i, uint32_t j) { return i == j ? pl.diag_slot : slot_of(i, j); }
inline uint32_t cell_slice(const Plan& pl, uint32_t i, uint32_t j) { return pl.full ? 0u : cell_slot(pl, i, j); }
// Byte offset of the cell's region (bpp bytes) from the start of j's allocation.
inline uint64_t cell_offset(const Plan& pl, uint32_t op, uint32_t i, uint32_t j) {
  return op == CDPROBE_OP_WRITE ? pl.land_off + (uint64_t)cell_slot(pl, i, j) * pl.bpp
                                : pl.src_off + (uint64_t)cell_slice(pl, i, j) * pl.bpp;
}
// What cell (issuer g, target j) of cdprobe_memcpy copies with op (CDPROBE_OP_READ: a pull, CDPROBE_OP_WRITE: a
// push) and where it lands (DESIGN §5n).  The source is a source slice: the one g reads from j, in j's allocation, for
// a pull; the one j reads from g, in g's own allocation, for a push.  Its word k is src_word(seed, src_rank,
// first_word + k).  The destination is the block of the sender (the slice's owner) in the receiver's exchange area,
// so the cells of one round never land on the same bytes.
struct MemcpyCell {
  uint32_t src_rank;    // whose allocation holds the source slice
  uint64_t src_off;     // the slice's byte offset in that allocation
  uint64_t first_word;  // the slice's first word in src_rank's source buffer
  uint32_t dst_rank;    // whose exchange area receives the copy
  uint64_t dst_off;     // the block's byte offset in that area
};
MemcpyCell memcpy_cell(const Plan& pl, uint32_t op, uint32_t g, uint32_t j);
// The hardware queues cdprobe_ce_alltoall needs on the most loaded device of a process whose n_local ranks run on
// ordinal[0 .. n_local) of an n-rank domain (diag: with a loop-back slice): each local rank holds its own stream and
// one copy stream per cell it issues, n - 1 peers and the diagonal.  *worst gets that device's ordinal (the lowest on
// a tie).  A stream wait blocks every stream that shares its queue, so the call needs at most
// CUDA_DEVICE_MAX_CONNECTIONS of them per device.
uint32_t ce_a2a_queues(uint32_t n, bool diag, uint32_t n_local, const int* ordinal, int* worst);
// Returns CDPROBE_OK or CDPROBE_ERR_ARG.
int make_plan(uint32_t n, uint64_t bytes, uint32_t mode, uint32_t flags, Plan* out);

}  // namespace cdp
