// topo.cc — node topology enumeration for the probe's caller (SURVEY.md §8f n2:
// "internal/common/topology.go").
//
// The north_star lists "internal/common topology enumeration" as a changing
// subsystem; the reference has none today (internal/common holds nvcap parsing
// only, SURVEY §2).  The daemon needs three facts before it opens a probe:
//   * which NVML index / UUID / PCI bus id each CUDA ordinal is (NVML and CUDA
//     enumerate in different orders unless CUDA_DEVICE_ORDER=PCI_BUS_ID),
//   * whether a GPU is in MIG mode (no P2P under MIG: identity matrix, H8),
//   * the node's clique id — "" on a single-node HGX box — with the exact
//     semantics of getCliqueIDStrict / getCliqueIDLegacy
//     (cmd/compute-domain-kubelet-plugin/nvlib.go:208-363), so the daemon and
//     the kubelet plugin agree on whether the IMEX gate applies.
// NVML is reached through nvml_loader.h.  No CUDA here; this file makes no
// reachability claim — reachability comes only from the kernels.
#include <stdio.h>
#include <string.h>

#include <set>
#include <string>

#include "../../include/cdprobe.h"
#include "nvml_loader.h"

namespace {

std::string hex_uuid(const unsigned char* b) {
  char s[40];
  snprintf(s, sizeof(s), "%02x%02x%02x%02x-%02x%02x-%02x%02x-%02x%02x-%02x%02x%02x%02x%02x%02x", b[0], b[1], b[2], b[3],
           b[4], b[5], b[6], b[7], b[8], b[9], b[10], b[11], b[12], b[13], b[14], b[15]);
  return s;
}

bool zero16(const unsigned char* b) {
  for (int i = 0; i < 16; ++i)
    if (b[i]) return false;
  return true;
}

}  // namespace

extern "C" int cdprobe_topology(uint32_t strict, cdprobe_topology_t* out) {
  if (out == nullptr) return CDPROBE_ERR_ARG;
  memset(out, 0, sizeof(*out));
  out->abi = CDPROBE_ABI_VERSION;
  cdp::Nvml nv;
  int rc = nv.open();
  if (rc != CDPROBE_OK) return rc;
  unsigned int n = 0;
  if (nv.count_(&n) != NVML_SUCCESS) return CDPROBE_ERR_CUDA;
  if (n > CDPROBE_MAX_GPUS) n = CDPROBE_MAX_GPUS;
  out->n = n;
  std::set<std::string> cluster_uuids, clique_ids;
  std::string first;
  for (unsigned int i = 0; i < n; ++i) {
    nvmlDevice_t d;
    if (nv.by_index_(i, &d) != NVML_SUCCESS) return CDPROBE_ERR_CUDA;
    if (nv.uuid_(d, out->uuid[i], sizeof(out->uuid[i])) != NVML_SUCCESS) return CDPROBE_ERR_CUDA;
    nvmlPciInfo_t pci;
    if (nv.pci_(d, &pci) == NVML_SUCCESS) snprintf(out->pci_bus_id[i], sizeof(out->pci_bus_id[i]), "%s", pci.busId);
    unsigned int cur = 0, pend = 0;
    out->mig[i] = (nv.mig_(d, &cur, &pend) == NVML_SUCCESS && cur == NVML_DEVICE_MIG_ENABLE) ? 1 : 0;
    for (unsigned int l = 0; l < CDPROBE_NVLINK_MAX_LINKS; ++l) {
      nvmlEnableState_t st = NVML_FEATURE_DISABLED;
      if (nv.link_(d, l, &st) == NVML_SUCCESS && st == NVML_FEATURE_ENABLED) {
        out->links_active[i]++;
        out->link_mask[i] |= 1u << l;
      }
    }
    if (out->clique_error[0] != '\0') continue;  // keep enumerating, the clique verdict is already an error
    nvmlGpuFabricInfo_t fi;
    memset(&fi, 0, sizeof(fi));
    const nvmlReturn_t fr = nv.fabric_(d, &fi);
    if (fr == NVML_ERROR_NOT_SUPPORTED) continue;  // no-clique fallback, nvlib.go:294-297
    if (fr != NVML_SUCCESS) {
      snprintf(out->clique_error, sizeof(out->clique_error), "failed to get GPU fabric info (device %u)", i);
      continue;
    }
    out->fabric_state[i] = fi.state;
    if (strict) {
      if (fi.state == NVML_GPU_FABRIC_STATE_NOT_SUPPORTED) continue;
      if (fi.state != NVML_GPU_FABRIC_STATE_COMPLETED) {
        snprintf(out->clique_error, sizeof(out->clique_error),
                 "NVLink fabric not attached (device %u): state=%u, refusing to start", i, (unsigned)fi.state);
        continue;
      }
      if (fi.status != NVML_SUCCESS) {
        snprintf(out->clique_error, sizeof(out->clique_error),
                 "NVLink fabric registration error (device %u): status=%d, refusing to start", i, (int)fi.status);
        continue;
      }
      if (zero16(fi.clusterUuid)) continue;  // NVLink-capable, not MNNVL-capable: nvlib.go:320-323
    } else if (fi.state != NVML_GPU_FABRIC_STATE_COMPLETED || zero16(fi.clusterUuid) || fi.status != NVML_SUCCESS) {
      continue;  // IsFabricAttached() == false: go-nvlib device.go:268-289
    }
    const std::string cu = hex_uuid(fi.clusterUuid), cq = std::to_string(fi.cliqueId);
    if (cluster_uuids.empty()) first = cu + "." + cq;
    cluster_uuids.insert(cu);
    clique_ids.insert(cq);
  }
  if (out->clique_error[0] == '\0' && !cluster_uuids.empty()) {
    if (cluster_uuids.size() != 1)
      snprintf(out->clique_error, sizeof(out->clique_error), "unexpected number of unique ClusterUUIDs found on devices");
    else if (clique_ids.size() != 1)
      snprintf(out->clique_error, sizeof(out->clique_error), "unexpected number of unique CliqueIDs found on devices");
    else
      snprintf(out->clique_id, sizeof(out->clique_id), "%s", first.c_str());
  }
  return CDPROBE_OK;
}
