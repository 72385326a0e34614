// links.cc — the NVML side of CDPROBE_OPT_LINK_COUNTERS (DESIGN §5o): one sample of every local device's per-link
// counters, and the difference of two.  The payload they are reported next to is schedule.cc's link_payload.
#include "links.h"

#include <string.h>

namespace cdp {

namespace {

// Field f of link l is entry l * kLinkFields + f of the one nvmlDeviceGetFieldValues call per device and sample.
// The DL error fields are Hopper's per-link counters; nvml.h marks them unsupported from Blackwell on.
constexpr unsigned kFieldId[kLinkFields] = {NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_TX, NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_RX,
                                            NVML_FI_DEV_NVLINK_ERROR_DL_REPLAY, NVML_FI_DEV_NVLINK_ERROR_DL_RECOVERY,
                                            NVML_FI_DEV_NVLINK_ERROR_DL_CRC};

int32_t status_of(nvmlReturn_t r) { return r == NVML_ERROR_NOT_SUPPORTED ? CDPROBE_ERR_UNSUPPORTED : (int32_t)r; }

bool value_of(const nvmlFieldValue_t& v, uint64_t* out) {
  switch (v.valueType) {
    case NVML_VALUE_TYPE_UNSIGNED_LONG_LONG: *out = v.value.ullVal; return true;
    case NVML_VALUE_TYPE_UNSIGNED_LONG: *out = v.value.ulVal; return true;
    case NVML_VALUE_TYPE_UNSIGNED_INT: *out = v.value.uiVal; return true;
    case NVML_VALUE_TYPE_SIGNED_LONG_LONG: *out = (uint64_t)v.value.sllVal; return true;
    case NVML_VALUE_TYPE_SIGNED_INT: *out = (uint64_t)(int64_t)v.value.siVal; return true;
    default: return false;
  }
}

}  // namespace

void LinkSampler::open(uint32_t n, const char (*uuid)[48], const bool* mig) {
  n_ = n > CDPROBE_MAX_GPUS ? CDPROBE_MAX_GPUS : n;
  nvmlReturn_t init_rc = NVML_SUCCESS;
  const int rc = nv_.open(&init_rc);
  if (rc == CDPROBE_OK && nv_.by_uuid_ && nv_.fields_) nvml_status_ = 0;
  else if (rc == CDPROBE_ERR_NO_DEVICE && init_rc != NVML_SUCCESS) nvml_status_ = status_of(init_rc);
  else nvml_status_ = CDPROBE_ERR_UNSUPPORTED;  // no library, or one without the entry points the counters need
  for (uint32_t d = 0; d < n_; ++d) {
    status_[d] = nvml_status_;
    if (status_[d] != 0) continue;
    if (mig[d]) {  // a MIG instance has no NVLink fields of its own
      status_[d] = CDPROBE_ERR_UNSUPPORTED;
      continue;
    }
    const nvmlReturn_t r = nv_.by_uuid_(uuid[d], &dev_[d]);
    if (r != NVML_SUCCESS) status_[d] = status_of(r);
  }
}

void LinkSampler::sample(LinkSample* out, bool remote) {
  for (uint32_t d = 0; d < n_; ++d) {
    LinkSample& s = out[d];
    s = LinkSample();
    s.status = status_[d];
    if (s.status != 0) continue;
    for (unsigned l = 0; l < (unsigned)kLinks; ++l) {
      nvmlEnableState_t st = NVML_FEATURE_DISABLED;
      if (nv_.link_(dev_[d], l, &st) == NVML_SUCCESS && st == NVML_FEATURE_ENABLED) s.link_mask |= 1u << l;
    }
    nvmlFieldValue_t v[kLinks * kLinkFields];
    memset(v, 0, sizeof(v));
    for (int l = 0; l < kLinks; ++l)
      for (int f = 0; f < kLinkFields; ++f) {
        v[l * kLinkFields + f].fieldId = kFieldId[f];
        v[l * kLinkFields + f].scopeId = (unsigned)l;
      }
    const nvmlReturn_t r = nv_.fields_(dev_[d], kLinks * kLinkFields, v);
    if (r != NVML_SUCCESS) {
      s.status = status_of(r);
      continue;
    }
    bool any = false;
    for (int l = 0; l < kLinks; ++l)
      for (int f = 0; f < kLinkFields; ++f) {
        const nvmlFieldValue_t& x = v[l * kLinkFields + f];
        if (x.nvmlReturn == NVML_SUCCESS && value_of(x, &s.value[l][f])) any = true;
        else s.failed[l] |= 1u << f;
        if (x.nvmlReturn != NVML_ERROR_NOT_SUPPORTED) any = true;
      }
    if (!any) {  // every field NOT_SUPPORTED: no NVLink on this GPU (a PCIe card)
      s.status = CDPROBE_ERR_UNSUPPORTED;
      continue;
    }
    if (remote && nv_.remote_pci_)
      for (unsigned l = 0; l < (unsigned)kLinks; ++l) {
        if (!((s.link_mask >> l) & 1u)) continue;
        nvmlPciInfo_t pci;
        memset(&pci, 0, sizeof(pci));
        if (nv_.remote_pci_(dev_[d], l, &pci) == NVML_SUCCESS) {
          static_assert(sizeof(s.remote_bus_id[l]) == NVML_DEVICE_PCI_BUS_ID_BUFFER_SIZE, "bus id size");
          memcpy(s.remote_bus_id[l], pci.busId, sizeof(s.remote_bus_id[l]));
          s.remote_bus_id[l][sizeof(s.remote_bus_id[l]) - 1] = '\0';
        }
      }
  }
}

void link_delta(const LinkSample& before, const LinkSample& after, cdprobe_link_device_t* out) {
  out->status = before.status != 0 ? before.status : after.status;
  out->link_mask = out->lost_mask = out->error_mask = 0;
  memset(out->tx_kib, 0, sizeof(out->tx_kib));
  memset(out->rx_kib, 0, sizeof(out->rx_kib));
  memset(out->errors, 0, sizeof(out->errors));
  memset(out->failed_fields, 0, sizeof(out->failed_fields));
  memset(out->remote_bus_id, 0, sizeof(out->remote_bus_id));
  if (out->status != 0) return;
  out->link_mask = before.link_mask;
  out->lost_mask = before.link_mask & ~after.link_mask;
  for (int l = 0; l < kLinks; ++l) {
    memcpy(out->remote_bus_id[l], before.remote_bus_id[l], sizeof(out->remote_bus_id[l]));
    out->failed_fields[l] = before.failed[l] | after.failed[l];
    uint64_t dv[kLinkFields];
    for (int f = 0; f < kLinkFields; ++f) {
      const bool ok = !((out->failed_fields[l] >> f) & 1u) && after.value[l][f] >= before.value[l][f];
      dv[f] = ok ? after.value[l][f] - before.value[l][f] : 0;
    }
    out->tx_kib[l] = dv[0];
    out->rx_kib[l] = dv[1];
    for (int k = 0; k < 3; ++k) {
      out->errors[l][k] = dv[2 + k];
      if (dv[2 + k] != 0) out->error_mask |= 1u << l;
    }
  }
}

}  // namespace cdp
