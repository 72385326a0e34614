// diagnose.h — host-callable launcher of the cell diagnosis in diagnose_kernels.cu (cdprobe_diagnose).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "probe_types.h"

namespace cdp {

constexpr int kDiagSamples = 16;

struct DiagSample {     // field for field cdprobe_diag_sample_t
  uint64_t offset, expected, observed, word, run_seq;
  uint32_t kind;
  int32_t rank;
};

// What both passes leave in device memory.  The host clears it before the first pass.
struct DiagOut {
  unsigned long long bad_words, bad_granules;
  unsigned long long first_bad_n;     // ~(lowest byte offset of a bad word); 0 = none
  unsigned long long last_bad;        // highest byte offset of a bad word
  unsigned long long kind_count[kDiagKinds];
  unsigned long long bit_flips[64];   // FLIP words only
  DiagSample sample[kDiagSamples];    // the min(16, bad_words) lowest offsets, in order
};

// Device scratch of one diagnosis of a region of n_bytes: the DiagOut, then one bad-word count per 16 KiB granule.
inline size_t diag_scratch_bytes(uint64_t n_bytes) {
  return sizeof(DiagOut) + (size_t)((n_bytes + kGranuleBytes - 1) / kGranuleBytes) * sizeof(uint32_t);
}

// Enqueues the diagnosis of `region` (spec.n_words words, 128-byte aligned, as mapped for the current device) on
// `stream`: clear the DiagOut at `scratch`, compare every word, then write the samples.  Returns a cudaError_t.
int diag_launch(const uint8_t* region, const DiagSpec& spec, void* scratch, int sm_count, cudaStream_t stream);

}  // namespace cdp
