// nvls_emulate.cuh — the two multicast instructions of allreduce_nvls_kernel in unicast form, so that the kernel can
// run as n ranks on one device (tests/nvls_emulate.py force-includes this header into a copy of
// allreduce_nvls_kernels.cu whose two multimem asm statements call these helpers instead).
//
// The members of the emulated multicast object are n equal areas, each an input half followed by an output half.  The
// tables below hold member m's input and output base; the multicast addresses the kernel is given are member 0's.
//
// What this models is the result of each instruction, and nothing else:
//   multimem.ld_reduce .add.u64   the wrapping sum of the word at that offset over every member's input;
//   multimem.st .v4               the 16 bytes stored at that offset into every member's output.
// It does not model their ordering against other accesses, their atomicity (the sum here is n separate loads, the
// store n separate stores), or fence.proxy.alias, which the kernel still issues and which orders nothing here, since
// every access goes through one unicast mapping.
#pragma once
#include <stdint.h>

#define NVLS_EMUL_MAX_MEMBERS 16

__constant__ uint32_t nvls_emul_n;
__constant__ uint64_t nvls_emul_in[NVLS_EMUL_MAX_MEMBERS];   // member m's input half
__constant__ uint64_t nvls_emul_out[NVLS_EMUL_MAX_MEMBERS];  // member m's output half

// multimem.ld_reduce.relaxed.sys.global.add.u64 at mc, an address in member 0's input half.
__device__ __forceinline__ uint64_t nvls_emul_ld_reduce(const void* mc) {
  const uint64_t off = (uint64_t)mc - nvls_emul_in[0];
  uint64_t s = 0;
  for (uint32_t m = 0; m < nvls_emul_n; ++m) {
    uint64_t v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(nvls_emul_in[m] + off) : "memory");
    s += v;
  }
  return s;
}

// multimem.st.relaxed.sys.global.v4.f32 of (w0, w1) at mc, an address in member 0's output half.
__device__ __forceinline__ void nvls_emul_st(void* mc, uint64_t w0, uint64_t w1) {
  const uint64_t off = (uint64_t)mc - nvls_emul_out[0];
  for (uint32_t m = 0; m < nvls_emul_n; ++m)
    asm volatile("st.relaxed.sys.global.v2.u64 [%0], {%1, %2};" ::"l"(nvls_emul_out[m] + off), "l"(w0), "l"(w1)
                 : "memory");
}
