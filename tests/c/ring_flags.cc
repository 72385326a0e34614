// ring_flags.cc — runs the ring helpers of probe_types.h that cdprobe_allreduce_ring's host and kernel use on cases
// given on stdin, for tests/test_allreduce_ring_cpu.py.
//
// One case per line, numbers in decimal:
//   F <call_seq> <k> <r> <phase>  prints ring_flag
//   O <n> <s_max> <u>             prints ring_flag_off(s_max, u), ring_flags_off(s_max) and ring_area_bytes(n, s_max)
//   G                             prints kRingFlagUnits and kRingOff
#include <stdio.h>

#include "probe_types.h"

int main() {
  char op;
  while (scanf(" %c", &op) == 1) {
    if (op == 'F') {
      unsigned long long call;
      unsigned k, r, phase;
      if (scanf("%llu %u %u %u", &call, &k, &r, &phase) != 4) return 1;
      printf("%u\n", cdp::ring_flag(call, k, r, phase));
    } else if (op == 'O') {
      unsigned n;
      unsigned long long s_max, u;
      if (scanf("%u %llu %llu", &n, &s_max, &u) != 3) return 1;
      printf("%llu %llu %llu\n", (unsigned long long)cdp::ring_flag_off(s_max, u),
             (unsigned long long)cdp::ring_flags_off(s_max), (unsigned long long)cdp::ring_area_bytes(n, s_max));
    } else if (op == 'G') {
      printf("%u %llu\n", cdp::kRingFlagUnits, (unsigned long long)cdp::kRingOff);
    } else {
      return 1;
    }
  }
  return 0;
}
