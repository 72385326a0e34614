// ce_a2a_host.cc — runs the host arithmetic of cdprobe_ce_alltoall (ce_a2a_queues, plan.h; ce_a2a_value and
// kCeA2aOff, probe_types.h) on cases given on stdin, for tests/test_ce_alltoall_cpu.py.
//
// One case per line, numbers in decimal:
//   Q <n> <diag> <n_local> <ordinal>...   prints ce_a2a_queues and the ordinal it names
//   V <call_seq> <k> <rep> <reps>         prints ce_a2a_value
//   O                                     prints kCeA2aOff, kNvlsOff, the lines' bytes and kCtrlBytes
#include <stdio.h>

#include "plan.h"

int main() {
  char op;
  while (scanf(" %c", &op) == 1) {
    if (op == 'Q') {
      unsigned n, diag, n_local;
      if (scanf("%u %u %u", &n, &diag, &n_local) != 3 || n_local > (unsigned)cdp::kMaxRanks) return 1;
      int ordinal[cdp::kMaxRanks], worst = -1;
      for (unsigned i = 0; i < n_local; ++i)
        if (scanf("%d", &ordinal[i]) != 1) return 1;
      const uint32_t need = cdp::ce_a2a_queues(n, diag != 0, n_local, ordinal, &worst);
      printf("%u %d\n", need, worst);
    } else if (op == 'V') {
      unsigned long long call;
      unsigned k, rep, reps;
      if (scanf("%llu %u %u %u", &call, &k, &rep, &reps) != 4) return 1;
      printf("%llu\n", (unsigned long long)cdp::ce_a2a_value(call, k, rep, reps));
    } else if (op == 'O') {
      printf("%llu %llu %llu %llu\n", (unsigned long long)cdp::kCeA2aOff, (unsigned long long)cdp::kNvlsOff,
             (unsigned long long)(cdp::kMaxRanks * sizeof(cdp::FlagLine)), (unsigned long long)cdp::kCtrlBytes);
    } else {
      return 1;
    }
  }
  return 0;
}
