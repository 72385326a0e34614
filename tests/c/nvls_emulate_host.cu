// nvls_emulate_host.cu — runs allreduce_nvls_kernel as n ranks on one device, with its two multicast instructions
// emulated (nvls_emulate.cuh), for tests/test_allreduce_nvls_emulated_gpu.py.  tests/nvls_emulate.py writes the
// kernel's copy as allreduce_nvls_emulated.cu and compiles this file, which includes it, into one shared library.
//
// Every rank gets what cdprobe_allreduce_nvls gives it (measure.cc: nvls_launch, ar_params, domain_lines, nvls_fault):
// a 2 x s_max NVLS area, input then output; a scratch of sizeof(ArScratch); and a zeroed control block whose kNvlsOff
// lines carry the domain barriers.  The input holds the probe's source pattern, src_word(seed, rank, k), which is what
// the product copies into it from the probe source.  The multicast addresses are member 0's halves.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "allreduce_nvls_emulated.cu"

namespace nvls_emul {
using namespace cdp;

constexpr uint64_t kCtrlLinesBytes = kNvlsOff + kMaxRanks * sizeof(FlagLine);
constexpr uint64_t kTimeoutNs = 20ull * 1000 * 1000 * 1000;  // a protocol mistake ends as an aborted row, not a hang

// One rank's row as nvls_emul_call returns it, in 64-bit words: (S, X), t_rel and t_end of every rep of every size,
// then per size the bad word count and the lowest bad byte offset (~0: none), then the abort word.
constexpr uint64_t kSR = (uint64_t)kBwMaxSizes * kRepSlots;
constexpr uint64_t kRowWords = 4 * kSR + 2 * kBwMaxSizes + 1;

char g_err[512];

int fail(const char* what, cudaError_t e) {
  snprintf(g_err, sizeof(g_err), "%s: %s", what, cudaGetErrorString(e));
  return (int)e;
}

__global__ void fill_src(uint64_t* in, uint64_t seed, uint32_t rank, uint64_t words) {
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < words; k += (uint64_t)gridDim.x * blockDim.x)
    in[k] = src_word(seed, rank, k);
}

// The emulated multicast object's members for a context of n ranks: one table per module, so every call loads its
// own context's before it launches.
cudaError_t set_members(uint32_t n, const uint64_t* in, const uint64_t* out) {
  cudaError_t e = cudaMemcpyToSymbol(nvls_emul_n, &n, sizeof(n));
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(nvls_emul_in, in, sizeof(uint64_t) * NVLS_EMUL_MAX_MEMBERS);
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(nvls_emul_out, out, sizeof(uint64_t) * NVLS_EMUL_MAX_MEMBERS);
  return e;
}

struct Rank {
  uint8_t* area = nullptr;  // input [0, s_max), output [s_max, 2 s_max)
  ArScratch* scratch = nullptr;
  uint8_t* ctrl = nullptr;
  cudaStream_t stream = nullptr;
  uint32_t grid = 0;
};
}  // namespace nvls_emul
using namespace nvls_emul;

struct NvlsEmul {
  uint32_t n = 0;
  uint64_t s_max = 0, seed = 0;
  Rank r[kMaxRanks];
  uint64_t in[NVLS_EMUL_MAX_MEMBERS] = {}, out[NVLS_EMUL_MAX_MEMBERS] = {};  // member m's input and output half
};

extern "C" {

const char* nvls_emul_error() { return g_err; }

// kBwMaxSizes, kRepSlots and the words of one row.
void nvls_emul_dims(uint64_t* out) {
  out[0] = kBwMaxSizes;
  out[1] = kRepSlots;
  out[2] = kRowWords;
}

// Device 0's multiprocessor count and its free and total memory.
int nvls_emul_device(uint64_t* out) {
  int sms = 0;
  size_t free_b = 0, total_b = 0;
  cudaError_t e = cudaSetDevice(0);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  if (e == cudaSuccess) e = cudaMemGetInfo(&free_b, &total_b);
  if (e != cudaSuccess) return fail("device", e);
  out[0] = (uint64_t)sms;
  out[1] = free_b;
  out[2] = total_b;
  return 0;
}

void nvls_emul_close(NvlsEmul* x) {
  if (x == nullptr) return;
  cudaSetDevice(0);
  for (uint32_t i = 0; i < x->n; ++i) {
    Rank& R = x->r[i];
    if (R.stream != nullptr) cudaStreamSynchronize(R.stream);
    cudaFree(R.area);
    cudaFree(R.scratch);
    cudaFree(R.ctrl);
    if (R.stream != nullptr) cudaStreamDestroy(R.stream);
  }
  delete x;
}

// n ranks on device 0, rank i with grids[i] CTAs; every CTA of every rank must be resident at once, since the ranks
// wait for each other inside their kernels.  Returns null with nvls_emul_error() set on failure.
NvlsEmul* nvls_emul_open(uint32_t n, const uint32_t* grids, uint64_t s_max, uint64_t seed) {
  g_err[0] = 0;
  uint64_t dev[3];
  if (n == 0 || n > (uint32_t)kMaxRanks || s_max == 0 || s_max % 16 != 0) {
    snprintf(g_err, sizeof(g_err), "open: bad n %u or s_max %llu", n, (unsigned long long)s_max);
    return nullptr;
  }
  if (nvls_emul_device(dev) != 0) return nullptr;
  uint64_t ctas = 0;
  for (uint32_t i = 0; i < n; ++i) ctas += grids[i];
  if (ctas > dev[0] || ctas == 0) {
    snprintf(g_err, sizeof(g_err), "open: %llu CTAs in all, %llu multiprocessors", (unsigned long long)ctas,
             (unsigned long long)dev[0]);
    return nullptr;
  }
  NvlsEmul* x = new NvlsEmul;
  x->n = n;
  x->s_max = s_max;
  x->seed = seed;
  for (uint32_t i = 0; i < n; ++i) {
    Rank& R = x->r[i];
    R.grid = grids[i];
    cudaError_t e = cudaMalloc(&R.area, 2 * s_max);
    if (e == cudaSuccess) e = cudaMalloc(&R.scratch, sizeof(ArScratch));
    if (e == cudaSuccess) e = cudaMalloc(&R.ctrl, kCtrlLinesBytes);
    if (e == cudaSuccess) e = cudaMemset(R.ctrl, 0, kCtrlLinesBytes);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&R.stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) {
      fill_src<<<1024, 256>>>(reinterpret_cast<uint64_t*>(R.area), seed, i, s_max / 8);
      e = cudaGetLastError();
    }
    if (e != cudaSuccess) {
      fail("open", e);
      nvls_emul_close(x);
      return nullptr;
    }
    x->in[i] = reinterpret_cast<uint64_t>(R.area);
    x->out[i] = reinterpret_cast<uint64_t>(R.area + s_max);
  }
  const cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    fail("open: fill", e);
    nvls_emul_close(x);
    return nullptr;
  }
  return x;
}

// One call of the ladder sizes[0 .. n_sizes) (the largest at most s_max), reps timed reps each.  The fault (mode, k,
// word; k = kArNoFault: none) goes to rank fault_rank, or when fault_rank < 0 to the word's owner, the rank
// cdprobe_allreduce_nvls gives it (twoshot_owner).  Every output is zeroed, then every rank is launched on its own
// stream before any is waited for.  rows gets n rows of kRowWords words.
int nvls_emul_call(NvlsEmul* x, const uint64_t* sizes, uint32_t n_sizes, uint32_t reps, int32_t fault_rank,
                   uint32_t fault_mode, uint32_t fault_k, uint64_t fault_word, uint64_t call_seq, uint64_t* rows) {
  g_err[0] = 0;
  if (n_sizes == 0 || n_sizes > kBwMaxSizes || reps > kMaxTimedReps || sizes[n_sizes - 1] > x->s_max) {
    snprintf(g_err, sizeof(g_err), "call: bad ladder or reps");
    return -1;
  }
  uint32_t owner = kArNoFault;
  if (fault_k != kArNoFault) {
    if (fault_k >= n_sizes || fault_word >= sizes[fault_k] / 8) {
      snprintf(g_err, sizeof(g_err), "call: the fault names no size or word");
      return -1;
    }
    owner = fault_rank >= 0 ? (uint32_t)fault_rank
                            : twoshot_owner((sizes[fault_k] + kUnitBytes - 1) / kUnitBytes, x->n,
                                            fault_word / (kUnitBytes / 8));
  }
  cudaError_t e = cudaSetDevice(0);
  if (e == cudaSuccess) e = set_members(x->n, x->in, x->out);  // another context may have been called since
  for (uint32_t i = 0; i < x->n && e == cudaSuccess; ++i) {
    e = cudaMemset(x->r[i].area + x->s_max, 0, x->s_max);
    if (e == cudaSuccess) e = cudaMemset(x->r[i].scratch, 0, sizeof(ArScratch));
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return fail("call: member tables and zero", e);
  for (uint32_t g = 0; g < x->n; ++g) {
    Rank& R = x->r[g];
    NvlsParams p;
    memset(&p, 0, sizeof(p));
    for (uint32_t j = 0; j < x->n; ++j) {  // domain_lines
      if (j == g) continue;
      p.dom.sig_out[j] = reinterpret_cast<uint64_t*>(x->r[j].ctrl + kNvlsOff + (uint64_t)g * sizeof(FlagLine));
      p.dom.sig_in[j] = reinterpret_cast<const uint64_t*>(R.ctrl + kNvlsOff + (uint64_t)j * sizeof(FlagLine));
    }
    p.dom.call_seq = call_seq;
    p.mc_in = x->r[0].area;
    p.mc_out = x->r[0].area + x->s_max;
    p.out = R.area + x->s_max;
    p.scratch = R.scratch;
    memcpy(p.size, sizes, sizeof(uint64_t) * n_sizes);
    p.seed = x->seed;
    p.timeout_ns = kTimeoutNs;
    p.fault_word = fault_word;
    p.fault_k = g == owner ? fault_k : kArNoFault;
    p.fault_mode = fault_mode;
    p.rank = g;
    p.n = x->n;
    p.n_sizes = n_sizes;
    p.reps = reps;
    e = (cudaError_t)allreduce_nvls_launch(p, R.grid, false, R.stream);
    if (e != cudaSuccess) return fail("call: launch", e);
  }
  for (uint32_t i = 0; i < x->n && e == cudaSuccess; ++i) e = cudaStreamSynchronize(x->r[i].stream);
  if (e != cudaSuccess) return fail("call: wait", e);
  static ArScratch s;
  for (uint32_t i = 0; i < x->n; ++i) {
    e = cudaMemcpy(&s, x->r[i].scratch, sizeof(s), cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) return fail("call: read back", e);
    uint64_t* row = rows + i * kRowWords;
    for (uint32_t k = 0; k < kBwMaxSizes; ++k)
      for (uint32_t r = 0; r < kRepSlots; ++r) {
        const uint64_t at = (uint64_t)k * kRepSlots + r;
        row[at] = s.rep.rep[k][r].sum;
        row[kSR + at] = s.rep.rep[k][r].xr;
        row[2 * kSR + at] = s.rep.t_rel[k][r];
        row[3 * kSR + at] = s.rep.rep[k][r].t_end;
      }
    for (uint32_t k = 0; k < kBwMaxSizes; ++k) {
      row[4 * kSR + k] = s.bad_words[k];
      row[4 * kSR + kBwMaxSizes + k] = ~s.first_bad_n[k];
    }
    row[4 * kSR + 2 * kBwMaxSizes] = s.rep.abort_flag;
  }
  return 0;
}

// Xors mask into word `word` of rank's input, at rest.
int nvls_emul_corrupt(NvlsEmul* x, uint32_t rank, uint64_t word, uint64_t mask) {
  g_err[0] = 0;
  if (rank >= x->n || word >= x->s_max / 8) {
    snprintf(g_err, sizeof(g_err), "corrupt: no rank %u word %llu", rank, (unsigned long long)word);
    return -1;
  }
  uint64_t* p = reinterpret_cast<uint64_t*>(x->r[rank].area) + word;
  uint64_t v = 0;
  cudaError_t e = cudaSetDevice(0);
  if (e == cudaSuccess) e = cudaMemcpy(&v, p, 8, cudaMemcpyDeviceToHost);
  v ^= mask;
  if (e == cudaSuccess) e = cudaMemcpy(p, &v, 8, cudaMemcpyHostToDevice);
  return e != cudaSuccess ? fail("corrupt", e) : 0;
}

}  // extern "C"
