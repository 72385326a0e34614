// bwcurve.h — host-callable launchers of the bandwidth-versus-size kernels in bwcurve_kernels.cu (cdprobe_bwcurve),
// and the layout of the scratch buffer they share with the host.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "probe_types.h"
#include "timed_rep.cuh"

namespace cdp {

constexpr uint32_t kBwDefaultReps = 8;

// The head of a local rank's scratch buffer during one bwcurve_kernel launch; the host zeroes it before each launch
// and reads it back after.  Rep r of size k (r = 0: the warm-up) ran from t_rel[k][r], the barrier leader's release
// stamp, to rep[k][r].t_end, the latest CTA completion stamp; rep[k][r].sum / xr is the (S, X) it read.
struct BwScratch {
  alignas(128) unsigned int abort_flag;  // set by the first CTA past the deadline; every CTA then stops
  alignas(128) unsigned int arrive;      // CTA arrivals at the grid barrier, over the whole launch
  alignas(128) unsigned long long release;  // grid barriers released so far
  alignas(128) unsigned long long t_rel[kBwMaxSizes][kRepSlots];
  Acc rep[kBwMaxSizes][kRepSlots];
};

struct BwCurveParams {
  const uint8_t* region;  // the cell's source slice through the issuer's mapping
  BwScratch* scratch;
  uint64_t size[kBwMaxSizes];  // the ladder (bwcurve_ladder)
  uint64_t timeout_ns;         // device deadline from kernel entry
  uint32_t n_sizes, reps;      // reps: timed reps (rep 0, the warm-up, comes on top)
  uint32_t path;               // ProbeParams::path
};

// Launches bwcurve_kernel on `stream` of the current device: `grid` CTAs of the probe kernel's shape, cooperative or
// not as the probe launches them.  For every size, one warm-up and p.reps timed reps, separated by grid barriers,
// each reading the first size bytes of p.region through the probe's read path p.path.  Returns a cudaError_t.
int bwcurve_launch(const BwCurveParams& p, unsigned grid, bool cooperative, cudaStream_t stream);
// Writes gsum[g] / gxor[g], the sum and the xor of the words of whole granule g, for the first n_granules granules of
// the region whose word k is word(k).  Defined for SrcRegionWord (a cell's source slice) and AllReduceWord (the
// all-reduce output).  Returns a cudaError_t.
template <typename Word>
int granules_launch(uint64_t* gsum, uint64_t* gxor, const Word& word, uint64_t n_granules, unsigned grid,
                    cudaStream_t stream);

}  // namespace cdp
