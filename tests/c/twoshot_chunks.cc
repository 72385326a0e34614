// twoshot_chunks.cc — runs the chunk partition of probe_types.h that cdprobe_allreduce_twoshot's host and kernel use on
// cases given on stdin, for tests/test_allreduce_twoshot_cpu.py.
//
// One case per line, numbers in decimal:
//   <units> <n>    prints <lo_0> <hi_0> ... <lo_n-1> <hi_n-1>, rank r's units [lo_r, hi_r)
#include <stdio.h>

#include "probe_types.h"

int main() {
  unsigned long long units;
  unsigned n;
  while (scanf("%llu %u", &units, &n) == 2) {
    for (unsigned r = 0; r < n; ++r) {
      uint64_t lo, hi;
      cdp::twoshot_chunk(units, n, r, &lo, &hi);
      printf("%llu %llu%s", (unsigned long long)lo, (unsigned long long)hi, r + 1 < n ? " " : "\n");
    }
  }
  return 0;
}
