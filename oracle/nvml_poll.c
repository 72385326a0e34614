/*
 * nvml_poll.c — the reference's CPU/NVML view of the node, restated in C.
 * TEST INFRASTRUCTURE ONLY (see cdoracle.h): the boolean oracle of the parity
 * tests and the timed CPU baseline of bench.py.  Never linked into
 * libcdprobe.so.
 *
 * Each step cites the reference code it follows (paths relative to the
 * reference root; the reference is Go over cgo -> dlopen("libnvidia-ml.so.1")):
 *
 *   library load   vendor/github.com/NVIDIA/go-nvml/pkg/nvml/lib.go:29-80
 *                  (lazy dlopen, RTLD_LAZY | RTLD_GLOBAL)
 *   init/shutdown  cmd/compute-domain-kubelet-plugin/nvlib.go:107-123
 *                  (nvmlInitWithFlags(NVML_INIT_FLAG_NO_GPUS), always Shutdown)
 *   device walk    vendor/github.com/NVIDIA/go-nvlib/pkg/nvlib/device/device.go:464-495
 *   enumerate      cmd/gpu-kubelet-plugin/nvlib.go:457-531 (getGpuInfo getters)
 *   clique id      cmd/compute-domain-kubelet-plugin/nvlib.go:208-363
 *   link state     vendor/.../go-nvml/pkg/nvml/device.go:1652-1661 (binding only; the
 *                  reference never calls it, SURVEY.md F1 — the poll itself is the
 *                  north_star's "nvmlDeviceGetNvLinkState CPU path")
 *   P2P status     vendor/.../go-nvml/pkg/nvml/device.go:281-285
 *   IMEX gate      cmd/compute-domain-daemon/main.go:435-459
 *   reach[i][j]    SURVEY.md §8(c) frozen definition.
 */
#define _GNU_SOURCE
#include <dlfcn.h>
#include <nvml.h>
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/wait.h>
#include <time.h>
#include <unistd.h>

#include "cdoracle.h"

typedef struct {
  void* dl;
  nvmlReturn_t (*InitWithFlags)(unsigned int);
  nvmlReturn_t (*Shutdown)(void);
  nvmlReturn_t (*DeviceGetCount)(unsigned int*);
  nvmlReturn_t (*DeviceGetHandleByIndex)(unsigned int, nvmlDevice_t*);
  nvmlReturn_t (*DeviceGetUUID)(nvmlDevice_t, char*, unsigned int);
  nvmlReturn_t (*DeviceGetMinorNumber)(nvmlDevice_t, unsigned int*);
  nvmlReturn_t (*DeviceGetName)(nvmlDevice_t, char*, unsigned int);
  nvmlReturn_t (*DeviceGetMemoryInfo)(nvmlDevice_t, nvmlMemory_t*);
  nvmlReturn_t (*DeviceGetPciInfo)(nvmlDevice_t, nvmlPciInfo_t*);
  nvmlReturn_t (*DeviceGetCudaComputeCapability)(nvmlDevice_t, int*, int*);
  nvmlReturn_t (*DeviceGetArchitecture)(nvmlDevice_t, nvmlDeviceArchitecture_t*);
  nvmlReturn_t (*DeviceGetBrand)(nvmlDevice_t, nvmlBrandType_t*);
  nvmlReturn_t (*SystemGetDriverVersion)(char*, unsigned int);
  nvmlReturn_t (*SystemGetCudaDriverVersion)(int*);
  nvmlReturn_t (*DeviceGetMigMode)(nvmlDevice_t, unsigned int*, unsigned int*);
  nvmlReturn_t (*DeviceGetNvLinkState)(nvmlDevice_t, unsigned int, nvmlEnableState_t*);
  nvmlReturn_t (*DeviceGetP2PStatus)(nvmlDevice_t, nvmlDevice_t, nvmlGpuP2PCapsIndex_t, nvmlGpuP2PStatus_t*);
  nvmlReturn_t (*DeviceGetGpuFabricInfo)(nvmlDevice_t, nvmlGpuFabricInfo_t*);
} nvml_t;

static double now_ms(void) {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return ts.tv_sec * 1e3 + ts.tv_nsec / 1e6;
}

static int load_nvml(nvml_t* n) {
  memset(n, 0, sizeof(*n));
  const char* path = getenv("CDORACLE_NVML_PATH"); /* tests point this at tests/fake_nvml */
  if (path == NULL || path[0] == '\0') path = "libnvidia-ml.so.1";
  n->dl = dlopen(path, RTLD_LAZY | RTLD_GLOBAL);
  if (n->dl == NULL) return -1;
#define SYM(field, name)                       \
  *(void**)(&n->field) = dlsym(n->dl, name);   \
  if (n->field == NULL) {                      \
    dlclose(n->dl);                            \
    return -2;                                 \
  }
  SYM(InitWithFlags, "nvmlInitWithFlags")
  SYM(Shutdown, "nvmlShutdown")
  SYM(DeviceGetCount, "nvmlDeviceGetCount_v2")
  SYM(DeviceGetHandleByIndex, "nvmlDeviceGetHandleByIndex_v2")
  SYM(DeviceGetUUID, "nvmlDeviceGetUUID")
  SYM(DeviceGetMinorNumber, "nvmlDeviceGetMinorNumber")
  SYM(DeviceGetName, "nvmlDeviceGetName")
  SYM(DeviceGetMemoryInfo, "nvmlDeviceGetMemoryInfo")
  SYM(DeviceGetPciInfo, "nvmlDeviceGetPciInfo_v3")
  SYM(DeviceGetCudaComputeCapability, "nvmlDeviceGetCudaComputeCapability")
  SYM(DeviceGetArchitecture, "nvmlDeviceGetArchitecture")
  SYM(DeviceGetBrand, "nvmlDeviceGetBrand")
  SYM(SystemGetDriverVersion, "nvmlSystemGetDriverVersion")
  SYM(SystemGetCudaDriverVersion, "nvmlSystemGetCudaDriverVersion")
  SYM(DeviceGetMigMode, "nvmlDeviceGetMigMode")
  SYM(DeviceGetNvLinkState, "nvmlDeviceGetNvLinkState")
  SYM(DeviceGetP2PStatus, "nvmlDeviceGetP2PStatus")
  SYM(DeviceGetGpuFabricInfo, "nvmlDeviceGetGpuFabricInfo")
#undef SYM
  return 0;
}

static void format_cluster_uuid(const unsigned char* b, char* out, size_t cap) {
  /* google/uuid String(): 8-4-4-4-12 lower-case hex (used by nvlib.go:236,325) */
  snprintf(out, cap, "%02x%02x%02x%02x-%02x%02x-%02x%02x-%02x%02x-%02x%02x%02x%02x%02x%02x", b[0], b[1], b[2], b[3],
           b[4], b[5], b[6], b[7], b[8], b[9], b[10], b[11], b[12], b[13], b[14], b[15]);
}

static int all_zero(const unsigned char* b, int n) {
  for (int i = 0; i < n; ++i)
    if (b[i]) return 0;
  return 1;
}

/* cmd/compute-domain-daemon/main.go:435-459: exec nvidia-imex-ctl -c /imexd/imexd.cfg -q and
 * require combined stdout/stderr == "READY\n". Returns 1 ready, 0 not ready. */
static int imex_ctl_ready(void) {
  const char* bin = getenv("CDORACLE_IMEX_CTL");
  if (bin == NULL || bin[0] == '\0') bin = "nvidia-imex-ctl";
  int pfd[2];
  if (pipe(pfd) != 0) return 0;
  pid_t pid = fork();
  if (pid < 0) return 0;
  if (pid == 0) {
    dup2(pfd[1], 1);
    dup2(pfd[1], 2);
    close(pfd[0]);
    close(pfd[1]);
    execlp(bin, bin, "-c", "/imexd/imexd.cfg", "-q", (char*)NULL);
    _exit(127);
  }
  close(pfd[1]);
  char buf[256];
  size_t got = 0;
  ssize_t k;
  while (got < sizeof(buf) - 1 && (k = read(pfd[0], buf + got, sizeof(buf) - 1 - got)) > 0) got += (size_t)k;
  buf[got] = '\0';
  close(pfd[0]);
  int st = 0;
  waitpid(pid, &st, 0);
  if (!WIFEXITED(st) || WEXITSTATUS(st) != 0) return 0;
  return strcmp(buf, "READY\n") == 0;
}

/* ---- optional N-thread variant of the two polls (SURVEY.md §8d: "single thread and an N-thread variant").
 * One worker per GPU; NVML is thread-safe but serialises most calls on the RM lock, so this is what "all the
 * host threads it can use" buys the reference path. ---- */
typedef struct {
  nvml_t* nv;
  nvmlDevice_t* dev;
  unsigned int count, i;
  cdoracle_nvml_t* out;
  uint32_t calls;
  int phase; /* 0 link poll, 1 P2P poll */
} worker_t;

static void poll_links_of(nvml_t* nv, nvmlDevice_t* dev, unsigned int i, cdoracle_nvml_t* out, uint32_t* calls) {
  unsigned int cur = 0, pend = 0;
  nvmlReturn_t ret = nv->DeviceGetMigMode(dev[i], &cur, &pend);
  (*calls)++;
  out->mig_enabled[i] = (ret == NVML_SUCCESS && cur == NVML_DEVICE_MIG_ENABLE) ? 1 : 0;
  out->n_links[i] = 0;
  for (unsigned int l = 0; l < CDORACLE_MAX_LINKS; ++l) {
    nvmlEnableState_t st = NVML_FEATURE_DISABLED;
    ret = nv->DeviceGetNvLinkState(dev[i], l, &st);
    (*calls)++;
    /* NOT_SUPPORTED / INVALID_ARGUMENT for absent links => inactive (SURVEY App. A) */
    const int active = (ret == NVML_SUCCESS && st == NVML_FEATURE_ENABLED);
    out->link_active[i][l] = (uint8_t)active;
    out->n_links[i] += (uint8_t)active;
  }
}

static void poll_p2p_of(nvml_t* nv, nvmlDevice_t* dev, unsigned int count, unsigned int i, cdoracle_nvml_t* out,
                        uint32_t* calls) {
  for (unsigned int j = 0; j < count; ++j) {
    if (i == j) continue;
    const nvmlGpuP2PCapsIndex_t idx[3] = {NVML_P2P_CAPS_INDEX_NVLINK, NVML_P2P_CAPS_INDEX_READ, NVML_P2P_CAPS_INDEX_WRITE};
    int32_t* dst[3] = {out->p2p_nvlink, out->p2p_read, out->p2p_write};
    for (int k = 0; k < 3; ++k) {
      nvmlGpuP2PStatus_t st = NVML_P2P_STATUS_UNKNOWN;
      nvmlReturn_t ret = nv->DeviceGetP2PStatus(dev[i], dev[j], idx[k], &st);
      (*calls)++;
      dst[k][i * CDORACLE_MAX_GPUS + j] = ret == NVML_SUCCESS ? (int32_t)st : -(int32_t)ret;
    }
  }
}

static void* worker_main(void* arg) {
  worker_t* w = (worker_t*)arg;
  if (w->phase == 0) poll_links_of(w->nv, w->dev, w->i, w->out, &w->calls);
  else poll_p2p_of(w->nv, w->dev, w->count, w->i, w->out, &w->calls);
  return NULL;
}

static uint32_t run_phase(nvml_t* nv, nvmlDevice_t* dev, unsigned int count, cdoracle_nvml_t* out, int phase, int threaded) {
  uint32_t calls = 0;
  if (!threaded || count < 2) {
    for (unsigned int i = 0; i < count; ++i) {
      if (phase == 0) poll_links_of(nv, dev, i, out, &calls);
      else poll_p2p_of(nv, dev, count, i, out, &calls);
    }
    return calls;
  }
  pthread_t th[CDORACLE_MAX_GPUS];
  worker_t w[CDORACLE_MAX_GPUS];
  for (unsigned int i = 0; i < count; ++i) {
    w[i] = (worker_t){nv, dev, count, i, out, 0, phase};
    pthread_create(&th[i], NULL, worker_main, &w[i]);
  }
  for (unsigned int i = 0; i < count; ++i) {
    pthread_join(th[i], NULL);
    calls += w[i].calls;
  }
  return calls;
}

int cdoracle_nvml_poll(uint32_t n_max, uint32_t flags, cdoracle_nvml_t* out) {
  nvml_t nv;
  memset(out, 0, sizeof(*out));
  out->imex_gate = -1;
  const double t_start = now_ms();
  int lrc = load_nvml(&nv);
  if (lrc != 0) return lrc;
  uint32_t calls = 0;
  nvmlReturn_t ret;
  int rc = 0;

  double t0 = now_ms();
  ret = nv.InitWithFlags(NVML_INIT_FLAG_NO_GPUS);
  calls++;
  out->init_ms = now_ms() - t0;
  if (ret != NVML_SUCCESS) {
    dlclose(nv.dl);
    return (int)ret;
  }

  /* ---- device walk -------------------------------------------------------------- */
  nvmlDevice_t dev[CDORACLE_MAX_GPUS];
  unsigned int count = 0;
  t0 = now_ms();
  ret = nv.DeviceGetCount(&count);
  calls++;
  if (ret != NVML_SUCCESS) {
    rc = (int)ret;
    goto done;
  }
  if (count > CDORACLE_MAX_GPUS) count = CDORACLE_MAX_GPUS;
  if (n_max != 0 && count > n_max) count = n_max;
  out->n = count;
  for (unsigned int i = 0; i < count; ++i) {
    ret = nv.DeviceGetHandleByIndex(i, &dev[i]);
    calls++;
    if (ret != NVML_SUCCESS) {
      rc = (int)ret;
      goto done;
    }
    ret = nv.DeviceGetUUID(dev[i], out->uuid[i], sizeof(out->uuid[i]));
    calls++;
    if (ret != NVML_SUCCESS) {
      rc = (int)ret;
      goto done;
    }
  }

  /* ---- enumerate leg (config 1): cmd/gpu-kubelet-plugin/nvlib.go:457-531 ---------- */
  if (!(flags & CDORACLE_FLAG_NO_ENUMERATE)) {
    for (unsigned int i = 0; i < count; ++i) {
      unsigned int minor = 0, cur = 0, pend = 0;
      nvmlMemory_t mem;
      nvmlPciInfo_t pci;
      nvmlDeviceArchitecture_t arch;
      nvmlBrandType_t brand;
      ret = nv.DeviceGetMinorNumber(dev[i], &minor);
      calls++;
      if (ret != NVML_SUCCESS) {
        rc = (int)ret;
        goto done;
      }
      out->minor[i] = (int32_t)minor;
      ret = nv.DeviceGetMigMode(dev[i], &cur, &pend); /* IsMigCapable / IsMigEnabled */
      calls++;
      if (ret != NVML_SUCCESS && ret != NVML_ERROR_NOT_SUPPORTED) {
        rc = (int)ret;
        goto done;
      }
      ret = nv.DeviceGetMemoryInfo(dev[i], &mem);
      calls++;
      if (ret == NVML_SUCCESS) out->memory_total[i] = mem.total;
      else if (ret != NVML_ERROR_NOT_SUPPORTED) { /* nvlib.go:478-487 */
        rc = (int)ret;
        goto done;
      }
      ret = nv.DeviceGetName(dev[i], out->name[i], sizeof(out->name[i]));
      calls++;
      if (ret != NVML_SUCCESS) {
        rc = (int)ret;
        goto done;
      }
      ret = nv.DeviceGetArchitecture(dev[i], &arch);
      calls++;
      if (ret != NVML_SUCCESS) {
        rc = (int)ret;
        goto done;
      }
      ret = nv.DeviceGetBrand(dev[i], &brand);
      calls++;
      if (ret != NVML_SUCCESS) {
        rc = (int)ret;
        goto done;
      }
      ret = nv.DeviceGetCudaComputeCapability(dev[i], &out->cc_major[i], &out->cc_minor[i]);
      calls++;
      if (ret != NVML_SUCCESS) {
        rc = (int)ret;
        goto done;
      }
      ret = nv.SystemGetDriverVersion(out->driver_version, sizeof(out->driver_version));
      calls++;
      if (ret != NVML_SUCCESS) {
        rc = (int)ret;
        goto done;
      }
      ret = nv.SystemGetCudaDriverVersion(&out->cuda_driver_version);
      calls++;
      if (ret != NVML_SUCCESS) {
        rc = (int)ret;
        goto done;
      }
      ret = nv.DeviceGetPciInfo(dev[i], &pci);
      calls++;
      /* NOT_SUPPORTED where the GPU sits behind a virtualised PCI layer: no bus id (as libcdprobe's topology
       * walk), the rest of the poll still answers */
      if (ret == NVML_SUCCESS) snprintf(out->pci_bus_id[i], sizeof(out->pci_bus_id[i]), "%s", pci.busId);
      else if (ret != NVML_ERROR_NOT_SUPPORTED) {
        rc = (int)ret;
        goto done;
      }
    }
  }
  out->enumerate_ms = now_ms() - t0;

  /* ---- fabric info + clique id: cmd/compute-domain-kubelet-plugin/nvlib.go:208-363 -- */
  t0 = now_ms();
  {
    char first_uuid[40] = "";
    uint32_t first_clique = 0;
    int have = 0, n_uuid = 0, n_clique = 0;
    for (unsigned int i = 0; i < count && out->clique_err == 0; ++i) {
      nvmlGpuFabricInfo_t fi;
      memset(&fi, 0, sizeof(fi));
      ret = nv.DeviceGetGpuFabricInfo(dev[i], &fi);
      calls++;
      out->fabric_ret[i] = (int32_t)ret;
      if (ret == NVML_ERROR_NOT_SUPPORTED) continue; /* no-clique fallback (nvlib.go:294-297; device.go:271-273) */
      if (ret != NVML_SUCCESS) {
        out->clique_err = (int32_t)ret;
        snprintf(out->clique_err_text, sizeof(out->clique_err_text), "failed to get GPU fabric info (device %u)", i);
        break;
      }
      out->fabric_state[i] = fi.state;
      out->fabric_status[i] = (int32_t)fi.status;
      out->fabric_clique[i] = fi.cliqueId;
      memcpy(out->cluster_uuid[i], fi.clusterUuid, 16);
      if (flags & CDORACLE_FLAG_LEGACY_CLIQUE) {
        /* IsFabricAttached (go-nvlib device.go:268-289): any of these => not attached, skip */
        if (fi.state != NVML_GPU_FABRIC_STATE_COMPLETED || all_zero(fi.clusterUuid, 16) || fi.status != NVML_SUCCESS)
          continue;
      } else {
        if (fi.state == NVML_GPU_FABRIC_STATE_NOT_SUPPORTED) continue; /* nvlib.go:303-306 */
        if (fi.state != NVML_GPU_FABRIC_STATE_COMPLETED) {             /* nvlib.go:309-311 */
          out->clique_err = -1;
          snprintf(out->clique_err_text, sizeof(out->clique_err_text),
                   "NVLink fabric not attached (device %u): state=%u, refusing to start", i, (unsigned)fi.state);
          break;
        }
        if (fi.status != NVML_SUCCESS) { /* nvlib.go:314-316 */
          out->clique_err = -2;
          snprintf(out->clique_err_text, sizeof(out->clique_err_text),
                   "NVLink fabric registration error (device %u): status=%d, refusing to start", i, (int)fi.status);
          break;
        }
        if (all_zero(fi.clusterUuid, 16)) continue; /* nvlib.go:320-323: NVLink-capable, not MNNVL */
      }
      char us[40];
      format_cluster_uuid(fi.clusterUuid, us, sizeof(us));
      if (!have) {
        snprintf(first_uuid, sizeof(first_uuid), "%s", us);
        first_clique = fi.cliqueId;
        have = 1;
        n_uuid = n_clique = 1;
      } else {
        if (strcmp(first_uuid, us) != 0) n_uuid++;
        if (first_clique != fi.cliqueId) n_clique++;
      }
    }
    if (out->clique_err == 0 && have) {
      if (n_uuid != 1) { /* nvlib.go:266-268,351-353 */
        out->clique_err = -3;
        snprintf(out->clique_err_text, sizeof(out->clique_err_text),
                 "unexpected number of unique ClusterUUIDs found on devices");
      } else if (n_clique != 1) {
        out->clique_err = -4;
        snprintf(out->clique_err_text, sizeof(out->clique_err_text),
                 "unexpected number of unique CliqueIDs found on devices");
      } else {
        snprintf(out->clique_id, sizeof(out->clique_id), "%s.%u", first_uuid, first_clique);
      }
    }
  }
  out->fabric_ms = now_ms() - t0;

  /* ---- MIG mode + NvLink state poll: N x 18 calls -------------------------------- */
  t0 = now_ms();
  calls += run_phase(&nv, dev, count, out, 0, (flags & CDORACLE_FLAG_THREADS) != 0);
  out->link_poll_ms = now_ms() - t0;

  /* ---- P2P status poll: N(N-1) x {NVLINK, READ, WRITE} ----------------------------- */
  t0 = now_ms();
  calls += run_phase(&nv, dev, count, out, 1, (flags & CDORACLE_FLAG_THREADS) != 0);
  out->p2p_poll_ms = now_ms() - t0;

  /* ---- IMEX gate (only when the node has a clique: main.go:436-439) ---------------- */
  t0 = now_ms();
  {
    const char* env_clique = getenv("CLIQUE_ID"); /* env contract: computedomain.go:164-169 */
    const int has_clique = (env_clique != NULL && env_clique[0] != '\0');
    if (has_clique && !(flags & CDORACLE_FLAG_NO_IMEX_CTL)) out->imex_gate = imex_ctl_ready();
  }
  out->imex_ms = now_ms() - t0;

  /* ---- frozen reachability definition (SURVEY.md §8c) ------------------------------- */
  for (unsigned int i = 0; i < count; ++i) {
    for (unsigned int j = 0; j < count; ++j) {
      const unsigned int c = i * CDORACLE_MAX_GPUS + j;
      if (i == j) {
        out->reach[c] = 1;
        continue;
      }
      int ok = !out->mig_enabled[i] && !out->mig_enabled[j] && out->n_links[i] > 0 && out->n_links[j] > 0 &&
               out->p2p_nvlink[c] == NVML_P2P_STATUS_OK && out->p2p_read[c] == NVML_P2P_STATUS_OK &&
               out->p2p_write[c] == NVML_P2P_STATUS_OK;
      if (out->imex_gate == 0) ok = 0; /* domain gate failed: nothing off-diagonal is reachable */
      out->reach[c] = (uint8_t)ok;
    }
  }

done:
  t0 = now_ms();
  nv.Shutdown(); /* alwaysShutdown, nvlib.go:118-123 */
  calls++;
  out->shutdown_ms = now_ms() - t0;
  out->nvml_calls = calls;
  dlclose(nv.dl);
  out->total_ms = now_ms() - t_start;
  return rc;
}
