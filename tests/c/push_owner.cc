// push_owner.cc — runs the push all-reduce helpers of probe_types.h that cdprobe_allreduce_push's host and kernel use
// on cases given on stdin, for tests/test_allreduce_push_cpu.py.
//
// One case per line, numbers in decimal:
//   C <units> <n>      checks twoshot_owner(units, n, u) against twoshot_chunk for every u < units; prints how many
//                      units it checked and the first u whose owner's chunk does not hold it (-1: none)
//   W <units> <n> <u>  prints twoshot_owner(units, n, u)
//   G                  prints kPushOff
#include <stdio.h>

#include "probe_types.h"

int main() {
  char op;
  while (scanf(" %c", &op) == 1) {
    if (op == 'C') {
      unsigned long long units;
      unsigned n;
      if (scanf("%llu %u", &units, &n) != 2) return 1;
      long long bad = -1;
      for (unsigned long long u = 0; u < units && bad < 0; ++u) {
        const uint32_t o = cdp::twoshot_owner(units, n, u);
        uint64_t lo, hi;
        cdp::twoshot_chunk(units, n, o, &lo, &hi);
        if (o >= n || u < lo || u >= hi) bad = (long long)u;
      }
      printf("%llu %lld\n", units, bad);
    } else if (op == 'W') {
      unsigned long long units, u;
      unsigned n;
      if (scanf("%llu %u %llu", &units, &n, &u) != 3) return 1;
      printf("%u\n", cdp::twoshot_owner(units, n, u));
    } else if (op == 'G') {
      printf("%llu\n", (unsigned long long)cdp::kPushOff);
    } else {
      return 1;
    }
  }
  return 0;
}
