// bwcurve_fold.cc — runs the size ladder and the expected-checksum fold of probe_types.h (what cdprobe_bwcurve's host
// uses) on cases given on stdin, for tests/test_bwcurve_cpu.py.  The per-granule table the fold reads is computed here
// as granules_kernel<SrcRegionWord> computes it on the GPU: the sum and the xor of the 2048 pattern words of each
// whole granule.
//
// One case per line, numbers in decimal:
//   L <bpp>                                            prints: <n> <size 0> ... <size n-1>   (n = 0: refused)
//   F <seed> <rank> <first_word> <region_words> <m> <w_0> ... <w_m-1>
//                                                      prints per prefix of w_k words: <S> <X>
#include <stdio.h>

#include <vector>

#include "probe_types.h"

int main() {
  char kind[2];
  while (scanf("%1s", kind) == 1) {
    if (kind[0] == 'L') {
      unsigned long long bpp;
      if (scanf("%llu", &bpp) != 1) return 1;
      uint64_t size[cdp::kBwMaxSizes];
      const uint32_t n = cdp::bwcurve_ladder(bpp, size);
      printf("%u", n);
      for (uint32_t k = 0; k < n; ++k) printf(" %llu", (unsigned long long)size[k]);
      printf("\n");
    } else {
      unsigned long long seed, first, words, m;
      unsigned rank;
      if (scanf("%llu %u %llu %llu %llu", &seed, &rank, &first, &words, &m) != 5) return 1;
      const uint64_t granules = words / cdp::kGranuleWords;
      std::vector<uint64_t> gsum(granules), gxor(granules);
      for (uint64_t g = 0; g < granules; ++g)
        for (uint64_t k = 0; k < cdp::kGranuleWords; ++k) {
          const uint64_t w = cdp::src_word(seed, rank, first + g * cdp::kGranuleWords + k);
          gsum[g] += w;
          gxor[g] ^= w;
        }
      for (unsigned long long e = 0; e < m; ++e) {
        unsigned long long n;
        if (scanf("%llu", &n) != 1 || n > words) return 1;
        uint64_t s, x;
        cdp::bwcurve_prefix_checksum(gsum.data(), gxor.data(), seed, rank, first, n, &s, &x);
        printf("%llu %llu%s", (unsigned long long)s, (unsigned long long)x, e + 1 < m ? " " : "\n");
      }
    }
  }
  return 0;
}
