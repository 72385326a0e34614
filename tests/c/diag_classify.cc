// diag_classify.cc — runs the diagnosis classifier of probe_types.h (the code cdprobe_diagnose's kernel and host
// use) on words given on stdin, for tests/test_diagnose_cpu.py, which builds them with the CPU oracle.
//
// One case per line, numbers in decimal:
//   read  <seed> <n_ranks> <target> <first_word> <n_words> <src_words> <k> <observed>
//   write <seed> <n_ranks> <issuer> <target> <run_seq> <n_words> <k> <observed>
// prints: <expected word k of the cell> <kind> <rank> <word> <run_seq>
#include <stdio.h>
#include <string.h>

#include "probe_types.h"

int main() {
  char op[16];
  unsigned long long a[8];
  while (scanf("%15s", op) == 1) {
    cdp::DiagSpec s;
    unsigned long long k, observed;
    if (strcmp(op, "read") == 0) {
      if (scanf("%llu %llu %llu %llu %llu %llu %llu %llu", &a[0], &a[1], &a[2], &a[3], &a[4], &a[5], &k, &observed) != 8)
        return 2;
      s = cdp::diag_read_spec(a[0], (uint32_t)a[1], (uint32_t)a[2], a[3], a[4], a[5]);
    } else if (strcmp(op, "write") == 0) {
      if (scanf("%llu %llu %llu %llu %llu %llu %llu %llu", &a[0], &a[1], &a[2], &a[3], &a[4], &a[5], &k, &observed) != 8)
        return 2;
      s = cdp::diag_write_spec(a[0], (uint32_t)a[1], (uint32_t)a[2], (uint32_t)a[3], a[4], a[5]);
    } else {
      return 2;
    }
    const cdp::DiagClass c = cdp::diag_classify(s, observed);
    printf("%llu %u %d %llu %llu\n", (unsigned long long)cdp::diag_expected(s, k), c.kind, c.rank,
           (unsigned long long)c.word, (unsigned long long)c.run_seq);
  }
  return 0;
}
