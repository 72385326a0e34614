// memcpy_cells.cc — runs the plan-side cell geometry of cdprobe_memcpy (memcpy_cell, plan.h) on cases given on stdin,
// for tests/test_memcpy_cpu.py.
//
// One case per line, numbers in decimal:
//   <n> <bytes> <mode> <flags> <op>   prints the plan's bytes_per_pair and round count, then one line per cell in the
//                                     order cdprobe_memcpy runs them (the tournament's rounds, then the loop-back round
//                                     when the plan has one; ranks in order within a round):
//                                     <round> <issuer> <target> <src_rank> <src_off - src_off of the plan> <first_word>
//                                     <dst_rank> <dst_off>
//                                     and a line "end"; "bad" when make_plan refuses the case.
#include <stdio.h>

#include "plan.h"

int main() {
  unsigned n, mode, flags, op;
  unsigned long long bytes;
  while (scanf("%u %llu %u %u %u", &n, &bytes, &mode, &flags, &op) == 5) {
    cdp::Plan pl;
    if (cdp::make_plan(n, bytes, mode, flags, &pl) != CDPROBE_OK) {
      printf("bad\n");
      continue;
    }
    const uint32_t rounds = pl.rounds + (pl.diag ? 1u : 0u);
    printf("%llu %u\n", (unsigned long long)pl.bpp, rounds);
    for (uint32_t r = 0; r < rounds; ++r) {
      for (uint32_t g = 0; g < n; ++g) {
        const int q = r < pl.rounds ? pl.partner[r][g] : (int)g;
        if (q < 0) continue;
        const cdp::MemcpyCell c = cdp::memcpy_cell(pl, op, g, (uint32_t)q);
        printf("%u %u %d %u %llu %llu %u %llu\n", r, g, q, c.src_rank, (unsigned long long)(c.src_off - pl.src_off),
               (unsigned long long)c.first_word, c.dst_rank, (unsigned long long)c.dst_off);
      }
    }
    printf("end\n");
  }
  return 0;
}
