// ll_flags.cc — runs the LL helpers of probe_types.h that cdprobe_allreduce_ll's host and kernel use on cases given on
// stdin, for tests/test_allreduce_ll_cpu.py.
//
// One case per line, numbers in decimal:
//   L <bpp>                       prints the LL ladder: <n_sizes> <size_0> ... (n_sizes 0: no ladder)
//   F <call_seq> <k> <r>          prints ll_flag
//   S <seed> <j> <flag>           prints ll_salt
//   O <p> <n> <s> <s_max> <w>     prints ll_slot and ll_area_bytes(n, s_max)
#include <stdio.h>

#include "probe_types.h"

int main() {
  char op;
  while (scanf(" %c", &op) == 1) {
    if (op == 'L') {
      unsigned long long bpp;
      if (scanf("%llu", &bpp) != 1) return 1;
      uint64_t size[cdp::kBwMaxSizes];
      const uint32_t n = cdp::ll_ladder(bpp, size);
      printf("%u", n);
      for (uint32_t k = 0; k < n; ++k) printf(" %llu", (unsigned long long)size[k]);
      printf("\n");
    } else if (op == 'F') {
      unsigned long long call;
      unsigned k, r;
      if (scanf("%llu %u %u", &call, &k, &r) != 3) return 1;
      printf("%u\n", cdp::ll_flag(call, k, r));
    } else if (op == 'S') {
      unsigned long long seed;
      unsigned j, flag;
      if (scanf("%llu %u %u", &seed, &j, &flag) != 3) return 1;
      printf("%llu\n", (unsigned long long)cdp::ll_salt(seed, j, flag));
    } else if (op == 'O') {
      unsigned p, n, s;
      unsigned long long s_max, w;
      if (scanf("%u %u %u %llu %llu", &p, &n, &s, &s_max, &w) != 5) return 1;
      printf("%llu %llu\n", (unsigned long long)cdp::ll_slot(p, n, s, s_max, w),
             (unsigned long long)cdp::ll_area_bytes(n, s_max));
    } else {
      return 1;
    }
  }
  return 0;
}
