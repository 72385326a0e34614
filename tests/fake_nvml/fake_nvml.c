/*
 * fake_nvml.c — a scriptable stand-in for libnvidia-ml.so.1 (test fixture).
 *
 * Pattern borrowed from the reference's CPU-only CI, which LD-preloads a mock
 * libnvidia-ml.so (hack/ci/mock-nvml/setup-mock-gpu.sh:70-115); this one is a
 * few dozen lines of C driven by a text scenario so the oracle's logic
 * (oracle/nvml_poll.c) can be tested without a GPU.
 *
 * Scenario file (env FAKE_NVML_SCENARIO), one directive per line:
 *   gpus N                       number of GPUs (default 8)
 *   links N                      active links per GPU (default 18)
 *   link_down G L                link L of GPU G inactive
 *   p2p G1 G2 KIND STATUS        KIND in {read,write,nvlink}; STATUS = nvmlGpuP2PStatus_t (ordered pair)
 *   mig G 0|1                    MIG mode of GPU G
 *   fabric G STATE STATUS CLIQUE UUIDHEX32   fabric info of GPU G
 *   fabric_all STATE STATUS CLIQUE UUIDHEX32
 *   unsupported WHAT             WHAT in {nvlink,p2p,fabric,mig}: calls return NOT_SUPPORTED
 *   fail WHAT RET                WHAT in {init,count,fabric}: return nvmlReturn_t RET
 *   uuid_reverse                 UUID numbering is the reverse of index order
 */
#include <nvml.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define MAXG 16
#define MAXL 18

static struct {
  int loaded;
  int gpus, links;
  unsigned char link_down[MAXG][MAXL];
  int p2p[3][MAXG][MAXG];
  int mig[MAXG];
  nvmlGpuFabricInfo_t fabric[MAXG];
  int unsup_nvlink, unsup_p2p, unsup_fabric, unsup_mig;
  int fail_init, fail_count, fail_fabric;
  int uuid_reverse;
  int inited;
} S;

static void parse_uuid(const char* hex, unsigned char out[16]) {
  memset(out, 0, 16);
  for (int i = 0; i < 16 && hex[2 * i] && hex[2 * i + 1]; ++i) {
    unsigned v = 0;
    sscanf(hex + 2 * i, "%2x", &v);
    out[i] = (unsigned char)v;
  }
}

static void load(void) {
  if (S.loaded) return;
  memset(&S, 0, sizeof(S));
  S.loaded = 1;
  S.gpus = 8;
  S.links = MAXL;
  for (int g = 0; g < MAXG; ++g) {
    S.fabric[g].state = NVML_GPU_FABRIC_STATE_COMPLETED; /* NVLink-capable, not MNNVL: zero cluster UUID */
    S.fabric[g].status = NVML_SUCCESS;
  }
  const char* path = getenv("FAKE_NVML_SCENARIO");
  if (!path) return;
  FILE* f = fopen(path, "r");
  if (!f) return;
  char line[256];
  while (fgets(line, sizeof(line), f)) {
    char a[32], b[64];
    int x, y, z, w;
    if (sscanf(line, "gpus %d", &x) == 1) S.gpus = x > MAXG ? MAXG : x;
    else if (sscanf(line, "links %d", &x) == 1) S.links = x > MAXL ? MAXL : x;
    else if (sscanf(line, "link_down %d %d", &x, &y) == 2) {
      if (x >= 0 && x < MAXG && y >= 0 && y < MAXL) S.link_down[x][y] = 1;
    } else if (sscanf(line, "p2p %d %d %31s %d", &x, &y, a, &z) == 4) {
      int k = !strcmp(a, "read") ? 0 : !strcmp(a, "write") ? 1 : 2;
      if (x >= 0 && x < MAXG && y >= 0 && y < MAXG) S.p2p[k][x][y] = z;
    } else if (sscanf(line, "mig %d %d", &x, &y) == 2) {
      if (x >= 0 && x < MAXG) S.mig[x] = y;
    } else if (sscanf(line, "fabric_all %d %d %d %63s", &y, &z, &w, b) == 4) {
      for (int g = 0; g < MAXG; ++g) {
        S.fabric[g].state = (unsigned char)y;
        S.fabric[g].status = (nvmlReturn_t)z;
        S.fabric[g].cliqueId = (unsigned)w;
        parse_uuid(b, S.fabric[g].clusterUuid);
      }
    } else if (sscanf(line, "fabric %d %d %d %d %63s", &x, &y, &z, &w, b) == 5) {
      if (x >= 0 && x < MAXG) {
        S.fabric[x].state = (unsigned char)y;
        S.fabric[x].status = (nvmlReturn_t)z;
        S.fabric[x].cliqueId = (unsigned)w;
        parse_uuid(b, S.fabric[x].clusterUuid);
      }
    } else if (sscanf(line, "unsupported %31s", a) == 1) {
      if (!strcmp(a, "nvlink")) S.unsup_nvlink = 1;
      if (!strcmp(a, "p2p")) S.unsup_p2p = 1;
      if (!strcmp(a, "fabric")) S.unsup_fabric = 1;
      if (!strcmp(a, "mig")) S.unsup_mig = 1;
    } else if (sscanf(line, "fail %31s %d", a, &x) == 2) {
      if (!strcmp(a, "init")) S.fail_init = x;
      if (!strcmp(a, "count")) S.fail_count = x;
      if (!strcmp(a, "fabric")) S.fail_fabric = x;
    } else if (!strncmp(line, "uuid_reverse", 12)) {
      S.uuid_reverse = 1;
    }
  }
  fclose(f);
}

static int idx_of(nvmlDevice_t d) { return (int)((size_t)d - 1); }

nvmlReturn_t nvmlInitWithFlags(unsigned int flags) {
  (void)flags;
  S.loaded = 0; /* re-read the scenario on every init so one process can run several */
  load();
  if (S.fail_init) return (nvmlReturn_t)S.fail_init;
  S.inited = 1;
  return NVML_SUCCESS;
}
nvmlReturn_t nvmlInit_v2(void) { return nvmlInitWithFlags(0); }
nvmlReturn_t nvmlShutdown(void) {
  S.inited = 0;
  return NVML_SUCCESS;
}
nvmlReturn_t nvmlDeviceGetCount_v2(unsigned int* n) {
  load();
  if (S.fail_count) return (nvmlReturn_t)S.fail_count;
  *n = (unsigned)S.gpus;
  return NVML_SUCCESS;
}
nvmlReturn_t nvmlDeviceGetHandleByIndex_v2(unsigned int i, nvmlDevice_t* d) {
  load();
  if ((int)i >= S.gpus) return NVML_ERROR_INVALID_ARGUMENT;
  *d = (nvmlDevice_t)(size_t)(i + 1);
  return NVML_SUCCESS;
}
nvmlReturn_t nvmlDeviceGetUUID(nvmlDevice_t d, char* buf, unsigned int len) {
  int i = idx_of(d);
  int u = S.uuid_reverse ? S.gpus - 1 - i : i;
  snprintf(buf, len, "GPU-%08x-fa4e-0000-0000-%012x", 0xb2000000u + (unsigned)u, (unsigned)u);
  return NVML_SUCCESS;
}
nvmlReturn_t nvmlDeviceGetMinorNumber(nvmlDevice_t d, unsigned int* m) {
  *m = (unsigned)idx_of(d);
  return NVML_SUCCESS;
}
nvmlReturn_t nvmlDeviceGetName(nvmlDevice_t d, char* buf, unsigned int len) {
  (void)d;
  snprintf(buf, len, "NVIDIA H100 80GB HBM3 (fake)");
  return NVML_SUCCESS;
}
nvmlReturn_t nvmlDeviceGetMemoryInfo(nvmlDevice_t d, nvmlMemory_t* m) {
  (void)d;
  m->total = 81559ull << 20;
  m->free = m->total;
  m->used = 0;
  return NVML_SUCCESS;
}
nvmlReturn_t nvmlDeviceGetPciInfo_v3(nvmlDevice_t d, nvmlPciInfo_t* p) {
  memset(p, 0, sizeof(*p));
  snprintf(p->busId, sizeof(p->busId), "00000000:%02X:00.0", 0x10 + idx_of(d));
  return NVML_SUCCESS;
}
nvmlReturn_t nvmlDeviceGetCudaComputeCapability(nvmlDevice_t d, int* major, int* minor) {
  (void)d;
  *major = 9;
  *minor = 0;
  return NVML_SUCCESS;
}
nvmlReturn_t nvmlDeviceGetArchitecture(nvmlDevice_t d, nvmlDeviceArchitecture_t* a) {
  (void)d;
  *a = NVML_DEVICE_ARCH_HOPPER;
  return NVML_SUCCESS;
}
nvmlReturn_t nvmlDeviceGetBrand(nvmlDevice_t d, nvmlBrandType_t* b) {
  (void)d;
  *b = NVML_BRAND_NVIDIA;
  return NVML_SUCCESS;
}
nvmlReturn_t nvmlSystemGetDriverVersion(char* buf, unsigned int len) {
  snprintf(buf, len, "580.159.00");
  return NVML_SUCCESS;
}
nvmlReturn_t nvmlSystemGetCudaDriverVersion(int* v) {
  *v = 13000;
  return NVML_SUCCESS;
}
nvmlReturn_t nvmlDeviceGetMigMode(nvmlDevice_t d, unsigned int* cur, unsigned int* pend) {
  if (S.unsup_mig) return NVML_ERROR_NOT_SUPPORTED;
  *cur = *pend = (unsigned)S.mig[idx_of(d)];
  return NVML_SUCCESS;
}
nvmlReturn_t nvmlDeviceGetNvLinkState(nvmlDevice_t d, unsigned int link, nvmlEnableState_t* st) {
  if (S.unsup_nvlink) return NVML_ERROR_NOT_SUPPORTED;
  if ((int)link >= S.links) return NVML_ERROR_INVALID_ARGUMENT;
  *st = S.link_down[idx_of(d)][link] ? NVML_FEATURE_DISABLED : NVML_FEATURE_ENABLED;
  return NVML_SUCCESS;
}
nvmlReturn_t nvmlDeviceGetP2PStatus(nvmlDevice_t a, nvmlDevice_t b, nvmlGpuP2PCapsIndex_t k, nvmlGpuP2PStatus_t* st) {
  if (S.unsup_p2p) return NVML_ERROR_NOT_SUPPORTED;
  int kk = k == NVML_P2P_CAPS_INDEX_READ ? 0 : k == NVML_P2P_CAPS_INDEX_WRITE ? 1 : 2;
  *st = (nvmlGpuP2PStatus_t)S.p2p[kk][idx_of(a)][idx_of(b)];
  return NVML_SUCCESS;
}
nvmlReturn_t nvmlDeviceGetGpuFabricInfo(nvmlDevice_t d, nvmlGpuFabricInfo_t* fi) {
  if (S.unsup_fabric) return NVML_ERROR_NOT_SUPPORTED;
  if (S.fail_fabric) return (nvmlReturn_t)S.fail_fabric;
  *fi = S.fabric[idx_of(d)];
  return NVML_SUCCESS;
}
const char* nvmlErrorString(nvmlReturn_t r) {
  (void)r;
  return "fake nvml error";
}
