// pingpong_words.cc — runs the pingpong word packing and digest of probe_types.h (the functions cdprobe_pingpong's
// kernel and host use) on cases given on stdin, for tests/test_pingpong_cpu.py, which restates them in Python.
//
// One case per line, numbers in decimal:
//   W <call_seq> <round> <leg> <rep> <trip> <echo>     prints: <word>
//   D <call_seq> <round> <leg> <trips> <reps> <fault>  prints: <digest of a clean leg, from pingpong_rep_digest>
//                                                              <digest the initiator receives, trip by trip, when the
//                                                               responder answers trip <fault> of rep 1 with the echo
//                                                               of the next trip (fault < 0: no fault)>
#include <stdio.h>

#include "probe_types.h"

int main() {
  char kind[2];
  while (scanf("%1s", kind) == 1) {
    if (kind[0] == 'W') {
      unsigned long long call, round, leg, rep, trip, echo;
      if (scanf("%llu %llu %llu %llu %llu %llu", &call, &round, &leg, &rep, &trip, &echo) != 6) return 1;
      printf("%llu\n", (unsigned long long)cdp::pingpong_word(call, (uint32_t)round, (uint32_t)leg, (uint32_t)rep,
                                                               (uint32_t)trip, (uint32_t)echo));
    } else {
      unsigned long long call, round, leg, trips, reps;
      long long fault;
      if (scanf("%llu %llu %llu %llu %llu %lld", &call, &round, &leg, &trips, &reps, &fault) != 6) return 1;
      uint64_t clean = 0, got = 0;
      for (uint32_t rep = 0; rep <= (uint32_t)reps; ++rep) {
        clean ^= cdp::pingpong_rep_digest(call, (uint32_t)round, (uint32_t)leg, rep, (uint32_t)trips);
        for (uint32_t trip = 0; trip < (uint32_t)trips; ++trip) {
          const bool skip = rep == 1 && (long long)trip == fault;
          got ^= cdp::pingpong_word(call, (uint32_t)round, (uint32_t)leg, rep, skip ? trip + 1 : trip, 1);
        }
      }
      printf("%llu %llu\n", (unsigned long long)clean, (unsigned long long)got);
    }
  }
  return 0;
}
