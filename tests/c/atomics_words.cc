// atomics_words.cc — runs the start values, digests and sums of probe_types.h (the functions cdprobe_atomics' kernels
// and host use) on cases given on stdin, for tests/test_atomics_cpu.py, which restates them in Python.
//
// One case per line, numbers in decimal:
//   S <call_seq> <kind> <rep>   prints: <atomics_start>
//   D <start> <total>           prints: <atomics_rep_digest> <atomics_rep_sum>
#include <stdio.h>

#include "probe_types.h"

int main() {
  char kind[2];
  while (scanf("%1s", kind) == 1) {
    if (kind[0] == 'S') {
      unsigned long long call, k, rep;
      if (scanf("%llu %llu %llu", &call, &k, &rep) != 3) return 1;
      printf("%llu\n", (unsigned long long)cdp::atomics_start(call, (uint32_t)k, (uint32_t)rep));
    } else {
      unsigned long long start, total;
      if (scanf("%llu %llu", &start, &total) != 2) return 1;
      printf("%llu %llu\n", (unsigned long long)cdp::atomics_rep_digest(start, total),
             (unsigned long long)cdp::atomics_rep_sum(start, total));
    }
  }
  return 0;
}
