// allreduce_fold.cc — runs the expected-checksum fold of probe_types.h that cdprobe_allreduce's host uses on cases
// given on stdin, for tests/test_allreduce_cpu.py.  The per-granule table the fold reads is computed here as
// allreduce_granules_kernel computes it on the GPU: the sum and the xor of the 2048 summed words of each whole granule.
//
// One case per line, numbers in decimal:
//   F <seed> <n> <output_words> <m> <w_0> ... <w_m-1>    prints per prefix of w_k words: <S> <X>
#include <stdio.h>

#include <vector>

#include "probe_types.h"

int main() {
  char kind[2];
  while (scanf("%1s", kind) == 1) {
    unsigned long long seed, words, m;
    unsigned n;
    if (kind[0] != 'F' || scanf("%llu %u %llu %llu", &seed, &n, &words, &m) != 4) return 1;
    const uint64_t granules = words / cdp::kGranuleWords;
    std::vector<uint64_t> gsum(granules), gxor(granules);
    for (uint64_t g = 0; g < granules; ++g)
      for (uint64_t k = 0; k < cdp::kGranuleWords; ++k) {
        const uint64_t w = cdp::allreduce_word(seed, n, g * cdp::kGranuleWords + k);
        gsum[g] += w;
        gxor[g] ^= w;
      }
    for (unsigned long long e = 0; e < m; ++e) {
      unsigned long long nw;
      if (scanf("%llu", &nw) != 1 || nw > words) return 1;
      uint64_t s, x;
      cdp::allreduce_prefix_checksum(gsum.data(), gxor.data(), seed, n, nw, &s, &x);
      printf("%llu %llu%s", (unsigned long long)s, (unsigned long long)x, e + 1 < m ? " " : "\n");
    }
  }
  return 0;
}
