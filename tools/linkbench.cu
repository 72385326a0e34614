// linkbench.cu — development microbenchmark (not product): what can one H100 NVLink-4 port carry,
// and which SM-side access shape gets closest?  The copy engine is timed next to the SM paths on the same
// buffers, so the SM figures can be read against the same-box ceiling.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo tools/linkbench.cu -o tools/linkbench
//   tools/linkbench [bytes] [reps]  > linkbench_n2.jsonl      (needs >= 2 GPUs with P2P)
//
// Every line of output is one JSON record:
//   {"name": ..., "dir": "uni"|"bidi", "bytes": per-GPU payload of ONE op, "gbps": [min, median, max], ...}
// Kernel variants are timed with %globaltimer inside the kernel (first CTA start -> last CTA end) after a
// host-released start flag, so launch skew between the two GPUs is not in the figure; the copy engine is
// timed with CUDA events.  gbps is per GPU per direction (payload bytes only).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include <algorithm>
#include <string>
#include <vector>

#define CK(x)                                                                              \
  do {                                                                                     \
    cudaError_t e_ = (x);                                                                  \
    if (e_ != cudaSuccess) {                                                               \
      fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_));  \
      exit(2);                                                                             \
    }                                                                                      \
  } while (0)

namespace {

struct Stamp {
  unsigned long long t0, t1, sink, pad;
};

__device__ __forceinline__ uint64_t gtimer() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t n) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(n) : "memory");
}
__device__ __forceinline__ void mbar_expect(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void bulk_store(void* dst, uint32_t src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_store_hint(void* dst, uint32_t src, uint32_t bytes, uint64_t pol) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(dst), "r"(src),
               "r"(bytes), "l"(pol)
               : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Every kernel: wait for the host start flag, stamp, do its job on [cta0, cta0+nctas), fence, stamp.
__device__ __forceinline__ void k_begin(volatile unsigned int* start, Stamp* st) {
  if (threadIdx.x == 0) {
    while (*start == 0u) {
    }
    atomicMin(&st->t0, (unsigned long long)gtimer());
  }
  __syncthreads();
}
__device__ __forceinline__ void k_end(Stamp* st, uint64_t sink) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    atomicMax(&st->t1, (unsigned long long)gtimer());
    if (sink == 0x1234567ull) st->sink = sink;
  }
}

// ------------------------------------------------------------------ ld/st paths ----
template <int VEC /*16 or 32*/, int UNROLL>
__device__ uint64_t read_ldg(const uint8_t* src, uint64_t bytes, uint32_t gthread, uint32_t nthreads) {
  uint64_t acc = 0;
  const uint64_t nvec = bytes / VEC;
  for (uint64_t v = gthread; v < nvec; v += (uint64_t)nthreads * UNROLL) {
    if (VEC == 16) {
      uint4 r[UNROLL];
#pragma unroll
      for (int k = 0; k < UNROLL; ++k) {
        const uint64_t i = v + (uint64_t)k * nthreads;
        r[k] = make_uint4(0, 0, 0, 0);
        if (i < nvec)
          asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                       : "=r"(r[k].x), "=r"(r[k].y), "=r"(r[k].z), "=r"(r[k].w)
                       : "l"(src + i * 16));
      }
#pragma unroll
      for (int k = 0; k < UNROLL; ++k) acc += (uint64_t)r[k].x + r[k].y + r[k].z + r[k].w;
    } else {
      uint32_t r[UNROLL][8];
#pragma unroll
      for (int k = 0; k < UNROLL; ++k) {
        const uint64_t i = v + (uint64_t)k * nthreads;
#pragma unroll
        for (int q = 0; q < 8; ++q) r[k][q] = 0;
        if (i < nvec)  // 32 contiguous bytes per thread as two 128-bit loads (sm_90 has no 256-bit access)
          asm volatile(
              "ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
              "ld.global.L1::no_allocate.v4.u32 {%4,%5,%6,%7}, [%8+16];"
              : "=r"(r[k][0]), "=r"(r[k][1]), "=r"(r[k][2]), "=r"(r[k][3]), "=r"(r[k][4]), "=r"(r[k][5]),
                "=r"(r[k][6]), "=r"(r[k][7])
              : "l"(src + i * 32));
      }
#pragma unroll
      for (int k = 0; k < UNROLL; ++k)
#pragma unroll
        for (int q = 0; q < 8; ++q) acc += r[k][q];
    }
  }
  return acc;
}

template <int VEC, int UNROLL, int CSHINT /*0 none, 1 .cs, 2 .wt*/>
__device__ void write_stg(uint8_t* dst, uint64_t bytes, uint32_t gthread, uint32_t nthreads) {
  const uint64_t nvec = bytes / VEC;
  uint32_t z = gthread * 2654435761u;
  for (uint64_t v = gthread; v < nvec; v += (uint64_t)nthreads * UNROLL) {
#pragma unroll
    for (int k = 0; k < UNROLL; ++k) {
      const uint64_t i = v + (uint64_t)k * nthreads;
      z += 0x9E3779B9u;
      if (i < nvec) {
        if (VEC == 16) {
          if (CSHINT == 1)
            asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(dst + i * 16), "r"(z), "r"(z ^ 1u), "r"(z ^ 2u),
                         "r"(z ^ 3u)
                         : "memory");
          else if (CSHINT == 2)
            asm volatile("st.global.wt.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(dst + i * 16), "r"(z), "r"(z ^ 1u), "r"(z ^ 2u),
                         "r"(z ^ 3u)
                         : "memory");
          else
            asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(dst + i * 16), "r"(z), "r"(z ^ 1u),
                         "r"(z ^ 2u), "r"(z ^ 3u)
                         : "memory");
        } else {
          asm volatile(
              "st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};\n\t"
              "st.global.L1::no_allocate.v4.u32 [%0+16], {%5,%6,%7,%8};" ::"l"(dst + i * 32), "r"(z),
              "r"(z ^ 1u), "r"(z ^ 2u), "r"(z ^ 3u), "r"(z ^ 4u), "r"(z ^ 5u), "r"(z ^ 6u), "r"(z ^ 7u)
              : "memory");
        }
      }
    }
  }
}

// ------------------------------------------------------------------ TMA bulk paths ----
// One warp owns STAGES stages of UNIT bytes.  smem: [warps][STAGES][UNIT] then mbarriers.
template <int UNIT, int STAGES>
__device__ uint64_t read_tma(uint8_t* smem, uint64_t* bars, const uint8_t* src, uint64_t bytes, uint32_t gwarp,
                             uint32_t nwarps, int warp, int lane, bool touch) {
  const uint32_t stage0 = smem_u32(smem) + warp * STAGES * UNIT;
  const uint32_t bar0 = smem_u32(bars) + warp * STAGES * 8;
  const uint64_t n_units = bytes / UNIT;
  uint64_t acc = 0;
  uint64_t u_issue = gwarp;
  uint32_t parity = 0;
#pragma unroll
  for (int s = 0; s < STAGES; ++s) {
    if (u_issue < n_units) {
      if (lane == 0) {
        mbar_expect(bar0 + 8 * s, UNIT);
        bulk_load(stage0 + s * UNIT, src + u_issue * UNIT, UNIT, bar0 + 8 * s);
      }
      u_issue += nwarps;
    }
  }
  int s = 0;
  for (uint64_t u = gwarp; u < n_units; u += nwarps) {
    while (!mbar_try(bar0 + 8 * s, (parity >> s) & 1u)) {
    }
    parity ^= 1u << s;
    if (touch) {
      for (uint32_t o = lane * 16; o < UNIT; o += 512) {
        uint4 v;
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(stage0 + s * UNIT + o));
        acc += (uint64_t)v.x + v.y + v.z + v.w;
      }
    }
    __syncwarp();
    if (u_issue < n_units) {
      if (lane == 0) {
        fence_async_smem();
        mbar_expect(bar0 + 8 * s, UNIT);
        bulk_load(stage0 + s * UNIT, src + u_issue * UNIT, UNIT, bar0 + 8 * s);
      }
      u_issue += nwarps;
    }
    s = (s + 1 == STAGES) ? 0 : s + 1;
  }
  return acc;
}

// gen: regenerate the stage contents for every unit (what the probe does); else store the same smem again.
template <int UNIT, int STAGES>
__device__ void write_tma(uint8_t* smem, uint8_t* dst, uint64_t bytes, uint32_t gwarp, uint32_t nwarps, int warp,
                          int lane, bool gen, bool hint) {
  const uint32_t stage0 = smem_u32(smem) + warp * STAGES * UNIT;
  const uint64_t n_units = bytes / UNIT;
  const uint64_t pol = policy_evict_first();
  uint32_t it = 0;
  int s = 0;
  uint32_t z = gwarp * 2654435761u + lane;
  for (uint64_t u = gwarp; u < n_units; u += nwarps, ++it) {
    if (it >= (uint32_t)STAGES && lane == 0) bulk_wait_read<STAGES - 1>();
    __syncwarp();
    if (gen || it < (uint32_t)STAGES) {
      for (uint32_t o = lane * 16; o < UNIT; o += 512) {
        z += 0x9E3779B9u;
        asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(stage0 + s * UNIT + o), "r"(z), "r"(z ^ 1u), "r"(z ^ 2u),
                     "r"(z ^ 3u)
                     : "memory");
      }
      fence_async_smem();
      __syncwarp();
    }
    if (lane == 0) {
      if (hint) bulk_store_hint(dst + u * UNIT, stage0 + s * UNIT, UNIT, pol);
      else bulk_store(dst + u * UNIT, stage0 + s * UNIT, UNIT);
      bulk_commit();
    }
    s = (s + 1 == STAGES) ? 0 : s + 1;
  }
  if (lane == 0) bulk_wait_all();
  __syncwarp();
}

enum Op : int { kOpRead = 1, kOpWrite = 2 };
enum Path : int { kLdst128 = 0, kLdst256 = 1, kTma = 2 };

struct Args {
  const uint8_t* rsrc;  // peer memory to read
  uint8_t* wdst;        // peer memory to write
  uint64_t bytes;       // per op
  int split;            // CTAs [0, split) run op A (write), [split, grid) op B (read); split = grid: all A; 0: all B
  int opA, opB;
  int flags;            // bit0 gen, bit1 hint, bit2 touch (read: fold the stage)
  volatile unsigned int* start;
  Stamp* st;
};

template <int PATH, int WARPS, int UNIT, int STAGES, int UNROLL, int CSHINT>
__global__ void __launch_bounds__(WARPS * 32, 1) k_link(const __grid_constant__ Args a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)WARPS * STAGES * UNIT);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if constexpr (PATH == kTma) if (lane == 0) {
    for (int s = 0; s < STAGES; ++s) mbar_init(smem_u32(bars) + (warp * STAGES + s) * 8, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  k_begin(a.start, a.st);
  const bool inA = (int)blockIdx.x < a.split;
  const int op = inA ? a.opA : a.opB;
  const uint32_t cta0 = inA ? 0 : a.split, nctas = inA ? a.split : gridDim.x - a.split;
  const uint32_t lcta = blockIdx.x - cta0;
  uint64_t acc = 0;
  if (op == kOpRead) {
    if constexpr (PATH == kTma)
      acc = read_tma<UNIT, STAGES>(smem, bars, a.rsrc, a.bytes, lcta * WARPS + warp, nctas * WARPS, warp, lane, a.flags & 4);
    else if constexpr (PATH == kLdst128)
      acc = read_ldg<16, UNROLL>(a.rsrc, a.bytes, lcta * WARPS * 32 + threadIdx.x, nctas * WARPS * 32);
    else
      acc = read_ldg<32, UNROLL>(a.rsrc, a.bytes, lcta * WARPS * 32 + threadIdx.x, nctas * WARPS * 32);
  } else if (op == kOpWrite) {
    if constexpr (PATH == kTma)
      write_tma<UNIT, STAGES>(smem, a.wdst, a.bytes, lcta * WARPS + warp, nctas * WARPS, warp, lane, a.flags & 1, a.flags & 2);
    else if constexpr (PATH == kLdst128)
      write_stg<16, UNROLL, CSHINT>(a.wdst, a.bytes, lcta * WARPS * 32 + threadIdx.x, nctas * WARPS * 32);
    else
      write_stg<32, UNROLL, 0>(a.wdst, a.bytes, lcta * WARPS * 32 + threadIdx.x, nctas * WARPS * 32);
  }
  k_end(a.st, acc);
}

struct Gpu {
  int dev;
  uint8_t *src, *land;
  Stamp* st;          // device
  cudaStream_t s;
  cudaEvent_t e0, e1;
};

struct Variant {
  std::string name;
  void (*fn)(const Args);
  int threads;
  size_t smem;
  int ctas_per_sm;
};

unsigned int* g_start_h = nullptr;  // mapped pinned
uint64_t g_bytes = 1ull << 30;
int g_reps = 7;
std::vector<Gpu> g;

template <int PATH, int WARPS, int UNIT, int STAGES, int UNROLL, int CSHINT>
Variant make(const char* name, int ctas_per_sm = 1) {
  Variant v;
  v.name = name;
  v.fn = k_link<PATH, WARPS, UNIT, STAGES, UNROLL, CSHINT>;
  v.threads = WARPS * 32;
  v.smem = PATH == kTma ? (size_t)WARPS * STAGES * UNIT + 1024 : 0;
  v.ctas_per_sm = ctas_per_sm;
  for (auto& d : g) {
    CK(cudaSetDevice(d.dev));
    CK(cudaFuncSetAttribute(v.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)v.smem));
  }
  return v;
}

struct Med {
  double mn, md, mx;
};
Med med(std::vector<double> v) {
  std::sort(v.begin(), v.end());
  return {v.front(), v[v.size() / 2], v.back()};
}

// Runs variant v on the GPUs in `who` (issuer -> peer = issuer ^ 1) with the given op mix.
void run_kernel(const Variant& v, const char* dir, std::vector<int> who, int opA, int opB, double fracA, int flags,
                uint64_t bytes, int ctas = 132, const char* extra = "") {
  std::vector<double> rd, wr, tms;
  const int grid = ctas * v.ctas_per_sm;
  int split = (int)(grid * fracA + 0.5);
  for (int rep = 0; rep < g_reps + 2; ++rep) {
    *g_start_h = 0;
    for (int i : who) {
      CK(cudaSetDevice(g[i].dev));
      Stamp init = {~0ull, 0ull, 0ull, 0ull};
      CK(cudaMemcpyAsync(g[i].st, &init, sizeof(init), cudaMemcpyHostToDevice, g[i].s));
      Args a;
      a.rsrc = g[i ^ 1].src;
      a.wdst = g[i ^ 1].land;
      a.bytes = bytes;
      a.split = split;
      a.opA = opA;
      a.opB = opB;
      a.flags = flags;
      unsigned int* dptr;
      CK(cudaHostGetDevicePointer((void**)&dptr, g_start_h, 0));
      a.start = dptr;
      a.st = g[i].st;
      v.fn<<<grid, v.threads, v.smem, g[i].s>>>(a);
      CK(cudaGetLastError());
    }
    // give every kernel time to become resident, then release
    struct timespec ts = {0, 300000};
    nanosleep(&ts, nullptr);
    __sync_synchronize();
    *(volatile unsigned int*)g_start_h = 1;
    double tmax = 0;
    for (int i : who) {
      CK(cudaSetDevice(g[i].dev));
      CK(cudaStreamSynchronize(g[i].s));
      Stamp st;
      CK(cudaMemcpy(&st, g[i].st, sizeof(st), cudaMemcpyDeviceToHost));
      const double t = (double)(st.t1 - st.t0);
      if (t > tmax) tmax = t;
    }
    if (rep >= 2) tms.push_back(tmax);
  }
  const Med m = med(tms);
  const bool hasA = split > 0 && opA, hasB = split < grid && opB;
  // payload per GPU per direction: egress = own writes + the peer's reads of my memory (bidi) -> for the
  // symmetric bidi case both directions carry (writes + reads); uni: write egress only / read ingress only.
  const double payload = (double)bytes * ((hasA ? 1 : 0) + (hasB ? 1 : 0));
  printf("{\"name\": \"%s\", \"dir\": \"%s\", \"bytes\": %llu, \"ops\": \"%s%s\", \"split\": %d, \"grid\": %d, \"flags\": %d, "
         "\"gbps_per_direction\": [%.1f, %.1f, %.1f], \"us\": [%.1f, %.1f, %.1f]%s}\n",
         v.name.c_str(), dir, (unsigned long long)bytes, hasA ? (opA == kOpWrite ? "W" : "R") : "",
         hasB ? (opB == kOpWrite ? "W" : "R") : "", split, grid, flags, payload / m.mx, payload / m.md, payload / m.mn,
         m.mn / 1e3, m.md / 1e3, m.mx / 1e3, extra);
  fflush(stdout);
}

void run_ce(const char* name, bool bidi, bool push, uint64_t bytes) {
  std::vector<double> tms;
  for (int rep = 0; rep < g_reps + 2; ++rep) {
    const int nd = bidi ? 2 : 1;
    for (int i = 0; i < nd; ++i) {
      const int srcg = i, dstg = i ^ 1;
      const int owner = push ? srcg : dstg;  // which GPU's stream (and copy engine) carries the copy
      CK(cudaSetDevice(g[owner].dev));
      CK(cudaEventRecord(g[owner].e0, g[owner].s));
      CK(cudaMemcpyPeerAsync(g[dstg].land, g[dstg].dev, g[srcg].src, g[srcg].dev, bytes, g[owner].s));
      CK(cudaEventRecord(g[owner].e1, g[owner].s));
    }
    double tmax = 0;
    for (int i = 0; i < nd; ++i) {
      const int owner = push ? i : (i ^ 1);
      CK(cudaSetDevice(g[owner].dev));
      CK(cudaEventSynchronize(g[owner].e1));
      float ms = 0;
      CK(cudaEventElapsedTime(&ms, g[owner].e0, g[owner].e1));
      if (ms > tmax) tmax = ms;
    }
    if (rep >= 2) tms.push_back(tmax * 1e6);
  }
  const Med m = med(tms);
  printf("{\"name\": \"%s\", \"dir\": \"%s\", \"bytes\": %llu, \"ops\": \"CE-%s\", \"gbps_per_direction\": [%.1f, %.1f, %.1f], "
         "\"us\": [%.1f, %.1f, %.1f]}\n",
         name, bidi ? "bidi" : "uni", (unsigned long long)bytes, push ? "push" : "pull", bytes / m.mx, bytes / m.md,
         bytes / m.mn, m.mn / 1e3, m.md / 1e3, m.mx / 1e3);
  fflush(stdout);
}

}  // namespace

int main(int argc, char** argv) {
  if (argc > 1) g_bytes = strtoull(argv[1], nullptr, 0);
  if (argc > 2) g_reps = atoi(argv[2]);
  const char* only = argc > 3 ? argv[3] : "";
  int nd = 0;
  CK(cudaGetDeviceCount(&nd));
  if (nd < 2) {
    fprintf(stderr, "linkbench needs 2 GPUs\n");
    return 3;
  }
  CK(cudaHostAlloc((void**)&g_start_h, 64, cudaHostAllocMapped | cudaHostAllocPortable));
  g.resize(2);
  for (int i = 0; i < 2; ++i) {
    g[i].dev = i;
    CK(cudaSetDevice(i));
    int can = 0;
    CK(cudaDeviceCanAccessPeer(&can, i, i ^ 1));
    if (!can) {
      fprintf(stderr, "no P2P %d -> %d\n", i, i ^ 1);
      return 3;
    }
    CK(cudaDeviceEnablePeerAccess(i ^ 1, 0));
    CK(cudaMalloc(&g[i].src, g_bytes));
    CK(cudaMalloc(&g[i].land, g_bytes));
    CK(cudaMalloc(&g[i].st, sizeof(Stamp)));
    CK(cudaMemset(g[i].src, 0x5a, g_bytes));
    CK(cudaMemset(g[i].land, 0, g_bytes));
    CK(cudaStreamCreateWithFlags(&g[i].s, cudaStreamNonBlocking));
    CK(cudaEventCreate(&g[i].e0));
    CK(cudaEventCreate(&g[i].e1));
    CK(cudaDeviceSynchronize());
  }
  const uint64_t B = g_bytes, S = 153391616ull / 32768 * 32768;  // the probe's bytes_per_pair at N = 8 (rounded to 32 KiB)
  auto want = [&](const char* tag) { return only[0] == 0 || strstr(only, tag) != nullptr; };

  if (want("ce")) {
    for (uint64_t b : {B, S}) {
      run_ce("copy-engine", false, true, b);
      run_ce("copy-engine", false, false, b);
      run_ce("copy-engine", true, true, b);
      run_ce("copy-engine", true, false, b);
    }
  }
  const std::vector<int> one = {0}, both = {0, 1};
  // --- writes ---
  if (want("w")) {
    struct TV {
      Variant v;
      int flags;
    };
    std::vector<TV> tv;
    tv.push_back({make<kTma, 8, 8192, 3, 1, 0>("tma w8 u8K s3 (r01 probe shape)"), 1});
    tv.push_back({make<kTma, 8, 8192, 3, 1, 0>("tma w8 u8K s3 nogen"), 0});
    tv.push_back({make<kTma, 8, 8192, 3, 1, 0>("tma w8 u8K s3 evict_first"), 1 | 2});
    tv.push_back({make<kTma, 4, 16384, 3, 1, 0>("tma w4 u16K s3"), 1});
    tv.push_back({make<kTma, 2, 32768, 3, 1, 0>("tma w2 u32K s3"), 1});
    tv.push_back({make<kTma, 4, 8192, 6, 1, 0>("tma w4 u8K s6"), 1});
    tv.push_back({make<kTma, 8, 4096, 6, 1, 0>("tma w8 u4K s6"), 1});
    tv.push_back({make<kTma, 8, 2048, 12, 1, 0>("tma w8 u2K s12"), 1});
    tv.push_back({make<kTma, 16, 4096, 3, 1, 0>("tma w16 u4K s3"), 1});
    tv.push_back({make<kTma, 1, 65536, 3, 1, 0>("tma w1 u64K s3"), 1});
    tv.push_back({make<kLdst128, 8, 0, 0, 4, 0>("stg128 unroll4"), 0});
    tv.push_back({make<kLdst128, 8, 0, 0, 16, 0>("stg128 unroll16"), 0});
    tv.push_back({make<kLdst128, 8, 0, 0, 8, 1>("stg128.cs unroll8"), 0});
    tv.push_back({make<kLdst128, 8, 0, 0, 8, 2>("stg128.wt unroll8"), 0});
    tv.push_back({make<kLdst256, 8, 0, 0, 4, 0>("stg256 unroll4"), 0});
    tv.push_back({make<kLdst256, 8, 0, 0, 8, 0>("stg256 unroll8"), 0});
    tv.push_back({make<kLdst256, 8, 0, 0, 8, 0>("stg256 unroll8 x4cta", 4), 0});
    tv.push_back({make<kLdst128, 8, 0, 0, 8, 0>("stg128 unroll8 x4cta", 4), 0});
    for (auto& t : tv) {
      run_kernel(t.v, "uni", one, kOpWrite, 0, 1.0, t.flags, B);
      run_kernel(t.v, "bidi", both, kOpWrite, 0, 1.0, t.flags, B);
    }
    // CTA count for the best-known shapes
    Variant t0 = make<kTma, 8, 8192, 3, 1, 0>("tma w8 u8K s3");
    for (int c : {16, 32, 64, 111}) run_kernel(t0, "uni", one, kOpWrite, 0, 1.0, 1, B, c);
    run_kernel(t0, "uni", one, kOpWrite, 0, 1.0, 1, S);
    run_kernel(t0, "bidi", both, kOpWrite, 0, 1.0, 1, S);
  }
  // --- reads ---
  if (want("r")) {
    struct TV {
      Variant v;
      int flags;
    };
    std::vector<TV> tv;
    tv.push_back({make<kTma, 8, 8192, 3, 1, 0>("tma w8 u8K s3 (r01 probe shape)"), 4});
    tv.push_back({make<kTma, 8, 8192, 3, 1, 0>("tma w8 u8K s3 notouch"), 0});
    tv.push_back({make<kTma, 4, 16384, 3, 1, 0>("tma w4 u16K s3"), 4});
    tv.push_back({make<kTma, 2, 32768, 3, 1, 0>("tma w2 u32K s3"), 4});
    tv.push_back({make<kTma, 4, 8192, 6, 1, 0>("tma w4 u8K s6"), 4});
    tv.push_back({make<kTma, 8, 4096, 6, 1, 0>("tma w8 u4K s6"), 4});
    tv.push_back({make<kTma, 8, 2048, 12, 1, 0>("tma w8 u2K s12"), 4});
    tv.push_back({make<kLdst128, 8, 0, 0, 16, 0>("ldg128 unroll16"), 0});
    tv.push_back({make<kLdst256, 8, 0, 0, 8, 0>("ldg256 unroll8"), 0});
    tv.push_back({make<kLdst256, 8, 0, 0, 8, 0>("ldg256 unroll8 x4cta", 4), 0});
    for (auto& t : tv) {
      run_kernel(t.v, "uni", one, 0, kOpRead, 0.0, t.flags, B);
      run_kernel(t.v, "bidi", both, 0, kOpRead, 0.0, t.flags, B);
    }
  }
  // --- fused round: write on the first CTAs, read on the rest, both GPUs at once ---
  if (want("f")) {
    Variant t0 = make<kTma, 8, 8192, 3, 1, 0>("fused tma w8 u8K s3");
    for (double f : {0.25, 0.4, 0.5, 0.6, 0.75}) {
      run_kernel(t0, "bidi", both, kOpWrite, kOpRead, f, 1 | 4, B);
    }
    run_kernel(t0, "uni", one, kOpWrite, kOpRead, 0.5, 1 | 4, B);  // one issuer, both directions loaded
    run_kernel(t0, "bidi", both, kOpWrite, kOpRead, 0.5, 1 | 4, S);
    Variant t1 = make<kLdst256, 8, 0, 0, 8, 0>("fused ldst256 unroll8");
    run_kernel(t1, "bidi", both, kOpWrite, kOpRead, 0.5, 0, B);
    // asymmetric: GPU 0 writes while GPU 1 reads -> all payload flows 0 -> 1 (one direction carries 2 streams)
  }
  return 0;
}
