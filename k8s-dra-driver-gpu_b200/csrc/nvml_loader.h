// nvml_loader.h — the library's one way to reach NVML, shared by topo.cc (cdprobe_topology) and links.cc (the link
// counters of CDPROBE_OPT_LINK_COUNTERS).
//
// NVML is reached the way go-nvml reaches it: lazy dlopen of libnvidia-ml.so.1, or of CDPROBE_NVML_PATH when set
// (vendor/github.com/NVIDIA/go-nvml/pkg/nvml/lib.go:29-80), nvmlInitWithFlags(NVML_INIT_FLAG_NO_GPUS) and an
// unconditional shutdown when the loader goes away (nvlib.go:107-123).  The entry points cdprobe_topology needs are
// required; the ones only the link counters use are optional (null when the library lacks them), so a library that
// serves cdprobe_topology still does.
#pragma once
#include <dlfcn.h>
#include <nvml.h>
#include <stdlib.h>

#include "../../include/cdprobe.h"

namespace cdp {

class Nvml {
 public:
  Nvml() = default;
  Nvml(const Nvml&) = delete;
  Nvml& operator=(const Nvml&) = delete;
  ~Nvml() {
    if (inited_ && shutdown_) shutdown_();
    if (dl_) dlclose(dl_);
  }
  // CDPROBE_ERR_NO_DEVICE: no library, or nvmlInit failed (*init_rc says how); CDPROBE_ERR_UNSUPPORTED: a required
  // entry point is missing.
  int open(nvmlReturn_t* init_rc = nullptr) {
    const char* path = getenv("CDPROBE_NVML_PATH");
    if (path == nullptr || *path == '\0') path = "libnvidia-ml.so.1";
    dl_ = dlopen(path, RTLD_LAZY | RTLD_GLOBAL);
    if (dl_ == nullptr) return CDPROBE_ERR_NO_DEVICE;
    bool ok = sym(init_, "nvmlInitWithFlags") && sym(shutdown_, "nvmlShutdown") &&
              sym(count_, "nvmlDeviceGetCount_v2") && sym(by_index_, "nvmlDeviceGetHandleByIndex_v2") &&
              sym(uuid_, "nvmlDeviceGetUUID") && sym(pci_, "nvmlDeviceGetPciInfo_v3") &&
              sym(mig_, "nvmlDeviceGetMigMode") && sym(link_, "nvmlDeviceGetNvLinkState") &&
              sym(fabric_, "nvmlDeviceGetGpuFabricInfo");
    if (!ok) return CDPROBE_ERR_UNSUPPORTED;
    sym(by_uuid_, "nvmlDeviceGetHandleByUUID");
    sym(fields_, "nvmlDeviceGetFieldValues");
    sym(remote_pci_, "nvmlDeviceGetNvLinkRemotePciInfo_v2");
    const nvmlReturn_t r = init_(NVML_INIT_FLAG_NO_GPUS);
    if (init_rc != nullptr) *init_rc = r;
    if (r != NVML_SUCCESS) return CDPROBE_ERR_NO_DEVICE;
    inited_ = true;
    return CDPROBE_OK;
  }

  nvmlReturn_t (*init_)(unsigned int) = nullptr;
  nvmlReturn_t (*shutdown_)(void) = nullptr;
  nvmlReturn_t (*count_)(unsigned int*) = nullptr;
  nvmlReturn_t (*by_index_)(unsigned int, nvmlDevice_t*) = nullptr;
  nvmlReturn_t (*uuid_)(nvmlDevice_t, char*, unsigned int) = nullptr;
  nvmlReturn_t (*pci_)(nvmlDevice_t, nvmlPciInfo_t*) = nullptr;
  nvmlReturn_t (*mig_)(nvmlDevice_t, unsigned int*, unsigned int*) = nullptr;
  nvmlReturn_t (*link_)(nvmlDevice_t, unsigned int, nvmlEnableState_t*) = nullptr;
  nvmlReturn_t (*fabric_)(nvmlDevice_t, nvmlGpuFabricInfo_t*) = nullptr;
  // optional: the link counters only
  nvmlReturn_t (*by_uuid_)(const char*, nvmlDevice_t*) = nullptr;
  nvmlReturn_t (*fields_)(nvmlDevice_t, int, nvmlFieldValue_t*) = nullptr;
  nvmlReturn_t (*remote_pci_)(nvmlDevice_t, unsigned int, nvmlPciInfo_t*) = nullptr;

 private:
  template <typename Fn>
  bool sym(Fn& fn, const char* name) {
    fn = reinterpret_cast<Fn>(dlsym(dl_, name));
    return fn != nullptr;
  }
  void* dl_ = nullptr;
  bool inited_ = false;
};

}  // namespace cdp
