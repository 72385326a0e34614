// diagnose_kernels.cu — sm_90a kernels of cdprobe_diagnose: a word-for-word diff of one cell's region against
// the pattern spec (probe_types.h), after a run.
//
// Pass 1 (compare) : every warp streams whole 16 KiB granules, 32 lanes x 8 x 16 B per batch with
//                    ld.global.nc.L1::no_allocate.v4, and compares each word with the pattern.  A clean batch
//                    costs one compare per word.  Only when __any_sync sees a mismatch does the warp park the
//                    batch in shared memory and classify its bad words (diag_classify), count them per kind,
//                    and add the bit-flip histogram of FLIP words with one ballot + __popc per flipped bit.
//                    Lane 0 writes the granule's bad-word count into the scratch buffer.
// Pass 2 (samples) : one CTA.  A block scan over the per-granule counts, starting at the first bad granule,
//                    finds the granules that hold the 16 lowest-offset bad words and how many bad words come
//                    before each.  A warp re-reads each such granule; a sample's index is that prefix plus its
//                    rank inside the granule (ballots), so the samples are the lowest offsets, in order, whatever
//                    the timing of pass 1.
//
// probe_kernels.cu is untouched: the probe kernel's code generation does not depend on this file.
#include <cuda_runtime.h>
#include <stdint.h>

#include "diagnose.h"

namespace cdp {
namespace {

constexpr int kDiagThreads = 256;
constexpr int kDiagWarps = kDiagThreads / 32;
constexpr int kBatch = 8;                                  // 16-byte loads in flight per lane
constexpr uint32_t kGranuleVecs = kGranuleBytes / 16;      // 1024: one warp-wide load covers 32 of them
constexpr int kBatches = (int)(kGranuleVecs / 32 / kBatch);  // 4 batches per granule
constexpr uint32_t kFull = 0xffffffffu;

__device__ __forceinline__ uint4 ldg_nc_v4(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ uint64_t lo64(const uint4& v) { return (uint64_t)v.x | ((uint64_t)v.y << 32); }
__device__ __forceinline__ uint64_t hi64(const uint4& v) { return (uint64_t)v.z | ((uint64_t)v.w << 32); }

template <bool kWrite>
__device__ __forceinline__ uint64_t expected(const DiagSpec& s, uint64_t k) {
  return kWrite ? write_word(s.cand[0].salt, k) : src_word(s.seed, s.target, s.first_word + k);
}

__device__ __forceinline__ unsigned long long warp_min(unsigned long long v) {
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long u = __shfl_xor_sync(kFull, v, o);
    v = u < v ? u : v;
  }
  return v;
}
__device__ __forceinline__ unsigned long long warp_max(unsigned long long v) {
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long u = __shfl_xor_sync(kFull, v, o);
    v = u > v ? u : v;
  }
  return v;
}

// ---- pass 1 ---------------------------------------------------------------------------------------------------
template <bool kWrite>
__global__ void __launch_bounds__(kDiagThreads, 2) diag_compare_kernel(const uint4* __restrict__ region,
                                                                    const __grid_constant__ DiagSpec s, DiagOut* out,
                                                                    uint32_t* gcount) {
  __shared__ uint4 park[kDiagWarps][kBatch][32];  // a batch with a mismatch, so the slow path can index it
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint64_t n_vecs = s.n_words / 2;
  const uint64_t n_gran = (s.n_words * 8 + kGranuleBytes - 1) / kGranuleBytes;
  uint32_t bad = 0, granules = 0, kind[kDiagKinds] = {}, flips_lo = 0, flips_hi = 0;
  unsigned long long first = ~0ull, last = 0;
  for (uint64_t g = (uint64_t)blockIdx.x * kDiagWarps + warp; g < n_gran; g += (uint64_t)gridDim.x * kDiagWarps) {
    uint32_t g_bad = 0;
    for (int b = 0; b < kBatches; ++b) {
      const uint64_t v0 = g * kGranuleVecs + (uint64_t)b * kBatch * 32 + lane;  // load i reads vector v0 + 32 i
      uint4 v[kBatch];
#pragma unroll
      for (int i = 0; i < kBatch; ++i)
        v[i] = v0 + 32 * i < n_vecs ? ldg_nc_v4(region + v0 + 32 * i) : make_uint4(0u, 0u, 0u, 0u);
      uint32_t mism = 0;  // bit 2i + h: word h of load i differs
#pragma unroll
      for (int i = 0; i < kBatch; ++i) {
        const uint64_t vi = v0 + 32 * i;
        if (vi < n_vecs) {
          mism |= (uint32_t)(lo64(v[i]) != expected<kWrite>(s, 2 * vi)) << (2 * i);
          mism |= (uint32_t)(hi64(v[i]) != expected<kWrite>(s, 2 * vi + 1)) << (2 * i + 1);
        }
      }
      if (!__any_sync(kFull, mism != 0)) continue;
      // ---- slow path: only batches with a bad word get here ----
#pragma unroll
      for (int i = 0; i < kBatch; ++i) park[warp][i][lane] = v[i];
      __syncwarp();
      for (int p = 0; p < 2 * kBatch; ++p) {  // warp-uniform: the ballots below need every lane
        const bool is_bad = (mism >> p) & 1u;
        if (!__any_sync(kFull, is_bad)) continue;
        uint64_t d = 0;  // flipped bits of a FLIP word
        if (is_bad) {
          const uint4 q = park[warp][p >> 1][lane];
          const uint64_t obs = (p & 1) ? hi64(q) : lo64(q);
          const uint64_t k = 2 * (v0 + 32 * (uint64_t)(p >> 1)) + (p & 1);
          const DiagClass c = diag_classify(s, obs);
#pragma unroll
          for (int j = 0; j < kDiagKinds; ++j) kind[j] += c.kind == (uint32_t)j;
          ++bad;
          ++g_bad;
          first = k < first ? k : first;
          last = k > last ? k : last;
          if (c.kind == kDiagFlip) d = obs ^ expected<kWrite>(s, k);
        }
        uint32_t m = __reduce_or_sync(kFull, (uint32_t)d);
        while (m) {
          const int bit = __ffs(m) - 1;
          m &= m - 1;
          const uint32_t n = __popc(__ballot_sync(kFull, (uint32_t)(d >> bit) & 1u));
          if (lane == (uint32_t)bit) flips_lo += n;
        }
        m = __reduce_or_sync(kFull, (uint32_t)(d >> 32));
        while (m) {
          const int bit = __ffs(m) - 1;
          m &= m - 1;
          const uint32_t n = __popc(__ballot_sync(kFull, (uint32_t)(d >> (32 + bit)) & 1u));
          if (lane == (uint32_t)bit) flips_hi += n;
        }
      }
      __syncwarp();
    }
    const uint32_t gb = __reduce_add_sync(kFull, g_bad);
    if (lane == 0) gcount[g] = gb;
    granules += gb != 0;
  }
  // one set of atomics per warp, and none from a clean warp
  const uint32_t wbad = __reduce_add_sync(kFull, bad);
  if (wbad == 0) return;
  first = warp_min(first);
  last = warp_max(last);
  uint32_t wkind[kDiagKinds];
#pragma unroll
  for (int j = 0; j < kDiagKinds; ++j) wkind[j] = __reduce_add_sync(kFull, kind[j]);
  if (lane == 0) {
    atomicAdd(&out->bad_words, (unsigned long long)wbad);
    atomicAdd(&out->bad_granules, (unsigned long long)granules);
    atomicMax(&out->first_bad_n, ~(first * 8ull));
    atomicMax(&out->last_bad, last * 8ull);
#pragma unroll
    for (int j = 0; j < kDiagKinds; ++j)
      if (wkind[j]) atomicAdd(&out->kind_count[j], (unsigned long long)wkind[j]);
  }
  if (flips_lo) atomicAdd(&out->bit_flips[lane], (unsigned long long)flips_lo);
  if (flips_hi) atomicAdd(&out->bit_flips[32 + lane], (unsigned long long)flips_hi);
}

// ---- pass 2 ---------------------------------------------------------------------------------------------------
template <bool kWrite>
__global__ void __launch_bounds__(kDiagThreads) diag_sample_kernel(const uint4* __restrict__ region,
                                                                   const __grid_constant__ DiagSpec s, DiagOut* out,
                                                                   const uint32_t* gcount) {
  __shared__ uint64_t s_gran[kDiagSamples];  // a granule that holds some of the first `want` bad words ...
  __shared__ uint32_t s_before[kDiagSamples];  // ... and how many bad words lie before it
  __shared__ uint32_t s_warp[kDiagWarps];
  __shared__ uint32_t s_n, s_total;
  const unsigned long long n_bad = out->bad_words;
  if (n_bad == 0) return;
  const uint32_t want = n_bad < (unsigned long long)kDiagSamples ? (uint32_t)n_bad : (uint32_t)kDiagSamples;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint64_t n_vecs = s.n_words / 2;
  const uint64_t n_gran = (s.n_words * 8 + kGranuleBytes - 1) / kGranuleBytes;
  if (threadIdx.x == 0) s_n = s_total = 0;
  __syncthreads();
  for (uint64_t g0 = (~out->first_bad_n) / kGranuleBytes;; g0 += kDiagThreads) {
    const uint64_t gi = g0 + threadIdx.x;
    const uint32_t c = gi < n_gran ? gcount[gi] : 0u;
    uint32_t x = c;  // inclusive scan over the CTA
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(kFull, x, o);
      if (lane >= (uint32_t)o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    uint32_t base = 0, total = 0;
    for (int w = 0; w < kDiagWarps; ++w) {
      base += w < (int)warp ? s_warp[w] : 0u;
      total += s_warp[w];
    }
    const uint32_t before = s_total + base + x - c;
    if (c != 0 && before < want) {  // at most `want` granules qualify: each holds one of the first `want` words
      const uint32_t e = atomicAdd(&s_n, 1u);
      s_gran[e] = gi;
      s_before[e] = before;
    }
    __syncthreads();
    if (threadIdx.x == 0) s_total += total;
    __syncthreads();
    if (s_total >= want || g0 + kDiagThreads >= n_gran) break;
  }
  for (uint32_t e = warp; e < s_n; e += kDiagWarps) {
    const uint64_t g = s_gran[e];
    uint32_t pos = s_before[e];
    for (uint32_t row = 0; row < kGranuleVecs / 32 && pos < want; ++row) {  // word order: row, lane, half
      const uint64_t vi = g * kGranuleVecs + row * 32 + lane;
      uint64_t w[2] = {0, 0};
      bool b[2] = {false, false};
      if (vi < n_vecs) {
        const uint4 v = ldg_nc_v4(region + vi);
        w[0] = lo64(v);
        w[1] = hi64(v);
        b[0] = w[0] != expected<kWrite>(s, 2 * vi);
        b[1] = w[1] != expected<kWrite>(s, 2 * vi + 1);
      }
      const uint32_t m0 = __ballot_sync(kFull, b[0]), m1 = __ballot_sync(kFull, b[1]);
      const uint32_t below = (1u << lane) - 1u;
      uint32_t r = pos + __popc(m0 & below) + __popc(m1 & below);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (b[h] && r < want) {
          const uint64_t k = 2 * vi + h;
          const DiagClass c = diag_classify(s, w[h]);
          DiagSample& o = out->sample[r];
          o.offset = k * 8;
          o.expected = expected<kWrite>(s, k);
          o.observed = w[h];
          o.word = c.word;
          o.run_seq = c.run_seq;
          o.kind = c.kind;
          o.rank = c.rank;
        }
        r += b[h];
      }
      pos += __popc(m0) + __popc(m1);
    }
  }
}

}  // namespace

int diag_launch(const uint8_t* region, const DiagSpec& spec, void* scratch, int sm_count, cudaStream_t stream) {
  DiagOut* out = static_cast<DiagOut*>(scratch);
  uint32_t* gcount = reinterpret_cast<uint32_t*>(out + 1);
  const uint4* r = reinterpret_cast<const uint4*>(region);
  cudaError_t e = cudaMemsetAsync(out, 0, sizeof(DiagOut), stream);
  if (e != cudaSuccess) return (int)e;
  const uint64_t n_gran = (spec.n_words * 8 + kGranuleBytes - 1) / kGranuleBytes;
  int per_sm = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(
      &per_sm, spec.is_write ? diag_compare_kernel<true> : diag_compare_kernel<false>, kDiagThreads, 0);
  if (e != cudaSuccess) return (int)e;
  uint64_t grid = (uint64_t)sm_count * (uint64_t)(per_sm > 0 ? per_sm : 1);
  const uint64_t need = (n_gran + kDiagWarps - 1) / kDiagWarps;
  if (grid > need) grid = need;
  if (spec.is_write) {
    diag_compare_kernel<true><<<(unsigned)grid, kDiagThreads, 0, stream>>>(r, spec, out, gcount);
    diag_sample_kernel<true><<<1, kDiagThreads, 0, stream>>>(r, spec, out, gcount);
  } else {
    diag_compare_kernel<false><<<(unsigned)grid, kDiagThreads, 0, stream>>>(r, spec, out, gcount);
    diag_sample_kernel<false><<<1, kDiagThreads, 0, stream>>>(r, spec, out, gcount);
  }
  return (int)cudaGetLastError();
}

}  // namespace cdp
