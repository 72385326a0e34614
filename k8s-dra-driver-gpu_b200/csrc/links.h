// links.h — per-link NVLink counters of the local devices, sampled through NVML around a probe pass (DESIGN §5o).
// Host only, no CUDA: tests build links.cc against a fake libnvidia-ml.so.1.
#pragma once
#include <stdint.h>

#include "../../include/cdprobe.h"
#include "nvml_loader.h"

namespace cdp {

constexpr int kLinks = CDPROBE_NVLINK_MAX_LINKS;
constexpr int kLinkFields = 5;  // per link: DATA_TX, DATA_RX, DL_REPLAY, DL_RECOVERY, DL_CRC (CDPROBE_LINK_FIELD_* bits)

// What one sample read of one device.
struct LinkSample {
  int32_t status = 0;                  // as cdprobe_link_device_t.status
  uint32_t link_mask = 0;              // links ENABLED
  uint64_t value[kLinks][kLinkFields] = {};
  uint32_t failed[kLinks] = {};        // bit f: field f of the link returned an error
  char remote_bus_id[kLinks][32] = {};
};

// NVML and one device handle per UUID, from open() until the sampler goes away.
class LinkSampler {
 public:
  // Loads NVML (once) and resolves each of the n UUIDs.  Never fails: a device that cannot be sampled keeps its
  // status, which every sample of it reports.
  void open(uint32_t n, const char (*uuid)[48], const bool* mig);
  // One sample of every device: link states, then all fields in one nvmlDeviceGetFieldValues call per device.
  // remote: also read each link's remote PCI bus id.
  void sample(LinkSample* out, bool remote);
  uint32_t n() const { return n_; }

 private:
  Nvml nv_;
  int32_t nvml_status_ = CDPROBE_ERR_UNSUPPORTED;
  uint32_t n_ = 0;
  nvmlDevice_t dev_[CDPROBE_MAX_GPUS] = {};
  int32_t status_[CDPROBE_MAX_GPUS] = {};
};

// What a handle keeps for CDPROBE_OPT_LINK_COUNTERS from the option's first enabling until close: the sampler over
// the distinct devices of the local ranks, the samples of the run in progress and the last report.
struct LinkCounters {
  LinkSampler sampler;
  LinkSample before[CDPROBE_MAX_GPUS], after[CDPROBE_MAX_GPUS];
  double before_ms = 0;
  cdprobe_links_t report = {};  // rows, in the order of the sampler's devices, get rank_mask and uuid when opened
};

// The device row of a pass from its two samples (pure): deltas of the counters, the link masks, the remote bus ids
// of the first sample.  status, link_mask and remote ids come from `before`; a field that failed in either sample
// reads 0 and is marked in failed_fields.  rank_mask, uuid and the expected payload are the caller's.
void link_delta(const LinkSample& before, const LinkSample& after, cdprobe_link_device_t* out);

}  // namespace cdp
