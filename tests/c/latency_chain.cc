// latency_chain.cc — runs the dependent-load chase of probe_types.h (the functions cdprobe_latency's kernel and host
// use) on cases given on stdin, for tests/test_latency_cpu.py, which restates the chase in Python.
//
// One case per line, numbers in decimal:
//   <seed> <issuer> <target> <first_word> <lines> <hops> <reps>
// prints: <digest over reps 0 .. reps> <first line of rep 0> <line after the last hop of rep reps>
#include <stdio.h>

#include "probe_types.h"

int main() {
  unsigned long long seed, i, j, first, lines, hops, reps;
  while (scanf("%llu %llu %llu %llu %llu %llu %llu", &seed, &i, &j, &first, &lines, &hops, &reps) == 7) {
    uint64_t digest = 0;
    for (uint32_t r = 0; r <= (uint32_t)reps; ++r)
      digest ^= cdp::latency_rep_digest(seed, (uint32_t)i, (uint32_t)j, first, lines, r, (uint32_t)hops);
    uint64_t line = cdp::latency_start(seed, (uint32_t)i, (uint32_t)j, (uint32_t)reps, lines);
    for (uint32_t h = 0; h < (uint32_t)hops; ++h)
      line = cdp::latency_next(cdp::src_word(seed, (uint32_t)j, first + cdp::kLineWords * line), h, lines);
    printf("%llu %llu %llu\n", (unsigned long long)digest,
           (unsigned long long)cdp::latency_start(seed, (uint32_t)i, (uint32_t)j, 0, lines), (unsigned long long)line);
  }
  return 0;
}
