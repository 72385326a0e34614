// handle.cc — the probe handle behind the C ABI (include/cdprobe.h): open and close, peer mappings, options, fault
// hooks and the run path.  The on-demand measurements are in measure.cc.
//
// Who calls this: the compute-domain-daemon's `run()` owns one handle for the
// life of the pod (reference: cmd/compute-domain-daemon/main.go:212-347; the
// cliqueID == "" branch main.go:244-250 is the single-node HGX case) and
// re-runs the probe on every daemon-set change; `check()` (main.go:435-459)
// only reads the cached verdict.  bench.py drives the same ABI with one process
// per GPU (world_size > 1).
//
// Threading: cdprobe_run launches one persistent kernel per local GPU from the
// calling thread (a launch is ~4 us; the first device barrier absorbs the
// skew) and then polls the pinned result rows the kernels write.  No thread
// survives a call.
#include <errno.h>
#include <fcntl.h>
#include <sched.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <unistd.h>

#include <algorithm>
#include <new>
#include <string>
#include <vector>

#include "handle.h"
#include "links.h"
#include "probe_launch.h"
#include "schedule.h"

namespace cdp {

static int fail_drv(const cdprobe* h, const char* what, CUresult r) {
  set_err(std::string(what) + ": " + h->drv.error_name(r));
  if (r == CUDA_ERROR_OUT_OF_MEMORY) return CDPROBE_ERR_NOMEM;
  if (r == CUDA_ERROR_NOT_SUPPORTED) return CDPROBE_ERR_UNSUPPORTED;
  return CDPROBE_ERR_CUDA;
}

static void format_uuid(const cudaUUID_t& u, bool mig, char out[48]) {
  const unsigned char* b = reinterpret_cast<const unsigned char*>(u.bytes);
  snprintf(out, 48, "%s-%02x%02x%02x%02x-%02x%02x-%02x%02x-%02x%02x-%02x%02x%02x%02x%02x%02x", mig ? "MIG" : "GPU",
           b[0], b[1], b[2], b[3], b[4], b[5], b[6], b[7], b[8], b[9], b[10], b[11], b[12], b[13], b[14], b[15]);
}

static bool imex_channel0_present() {
  int fd = ::open("/dev/nvidia-caps-imex-channels/channel0", O_RDONLY | O_CLOEXEC);
  if (fd < 0) return false;
  ::close(fd);
  return true;
}

// Pinned memory on device `ordinal`, exportable as handle type `ht`.
static CUmemAllocationProp alloc_prop(int ordinal, CUmemAllocationHandleType ht) {
  CUmemAllocationProp ap;
  memset(&ap, 0, sizeof(ap));
  ap.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  ap.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  ap.location.id = ordinal;
  ap.requestedHandleTypes = ht;
  return ap;
}

// Creates `bytes` of alloc_prop(ordinal, ht) memory in *hnd.
static CUresult create_alloc(const cdprobe* h, int ordinal, CUmemAllocationHandleType ht, size_t bytes,
                             CUmemGenericAllocationHandle* hnd) {
  const CUmemAllocationProp ap = alloc_prop(ordinal, ht);
  return h->drv.MemCreate(hnd, bytes, &ap, 0);
}

// Reserves `bytes` of address space aligned to `align`, maps `hnd` there and opens it to device `ordinal` for reading
// and writing.  On failure nothing of it is kept.
static CUresult map_range(const cdprobe* h, CUmemGenericAllocationHandle hnd, size_t bytes, size_t align, int ordinal,
                          CUdeviceptr* va) {
  CUresult r = h->drv.MemAddressReserve(va, bytes, align, 0, 0);
  if (r != CUDA_SUCCESS) return r;
  r = h->drv.MemMap(*va, bytes, 0, hnd, 0);
  if (r != CUDA_SUCCESS) {
    h->drv.MemAddressFree(*va, bytes);
    return r;
  }
  CUmemAccessDesc ad;
  memset(&ad, 0, sizeof(ad));
  ad.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  ad.location.id = ordinal;
  ad.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  r = h->drv.MemSetAccess(*va, bytes, &ad, 1);
  if (r != CUDA_SUCCESS) {
    h->drv.MemUnmap(*va, bytes);
    h->drv.MemAddressFree(*va, bytes);
  }
  return r;
}

static void unmap_range(const cdprobe* h, CUdeviceptr va, size_t bytes) {
  h->drv.MemUnmap(va, bytes);
  h->drv.MemAddressFree(va, bytes);
}

// Map rank j's allocation of m into local rank li's address space.
static int32_t map_peer(cdprobe* h, SharedAlloc& m, uint32_t li, uint32_t j) {
  LocalRank& L = h->lr[li];
  if (m.mapped[li][j]) return 0;
  CUmemGenericAllocationHandle hnd;
  if (j >= h->first && j < h->first + h->n_local) {
    hnd = m.own[j - h->first];
  } else if (m.has_import[j]) {
    hnd = m.imported[j];
  } else {
    return CDPROBE_ERR_RENDEZVOUS;
  }
  if (cudaSetDevice(L.ordinal) != cudaSuccess) return CDPROBE_ERR_CUDA;
  CUdeviceptr va = 0;
  const CUresult r = map_range(h, hnd, m.bytes, kVmmGranule, L.ordinal, &va);
  if (r != CUDA_SUCCESS) return (int32_t)r;
  m.va[li][j] = va;
  m.mapped[li][j] = true;
  return 0;
}

static void unmap_peer(cdprobe* h, SharedAlloc& m, uint32_t li, uint32_t j) {
  if (!m.mapped[li][j]) return;
  cudaSetDevice(h->lr[li].ordinal);
  unmap_range(h, m.va[li][j], m.bytes);
  m.va[li][j] = 0;
  m.mapped[li][j] = false;
}

// Unmaps m everywhere, releases its imports, then its local allocations and their fds, and leaves m as never created.
static void release_shared(cdprobe* h, SharedAlloc& m) {
  for (uint32_t li = 0; li < h->n_local; ++li) {
    if (h->lr[li].ordinal < 0) continue;
    for (uint32_t j = 0; j < (uint32_t)kMaxRanks; ++j) unmap_peer(h, m, li, j);
  }
  for (uint32_t j = 0; j < (uint32_t)kMaxRanks; ++j)
    if (m.has_import[j]) h->drv.MemRelease(m.imported[j]);
  for (uint32_t li = 0; li < h->n_local; ++li) {
    if (h->lr[li].ordinal < 0) continue;
    cudaSetDevice(h->lr[li].ordinal);
    if (m.has_own[li]) h->drv.MemRelease(m.own[li]);
    if (m.own_fd[li] >= 0) ::close(m.own_fd[li]);
  }
  m = SharedAlloc();
}

// Local rank li's allocation of m: m.bytes of its device's memory, exportable as the handle type chosen at open.
static int create_own(cdprobe* h, SharedAlloc& m, uint32_t li) {
  LocalRank& L = h->lr[li];
  CDP_RT(cudaSetDevice(L.ordinal));
  const CUmemAllocationHandleType ht = h->handle_type == 8u   ? CU_MEM_HANDLE_TYPE_FABRIC
                                       : h->handle_type == 1u ? CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR
                                                              : CU_MEM_HANDLE_TYPE_NONE;
  const CUmemAllocationProp ap = alloc_prop(L.ordinal, ht);
  size_t gran = 0;
  CUresult r = h->drv.MemGetAllocationGranularity(&gran, &ap, CU_MEM_ALLOC_GRANULARITY_MINIMUM);
  if (r != CUDA_SUCCESS) return fail_drv(h, "cuMemGetAllocationGranularity", r);
  if (gran == 0 || kVmmGranule % gran != 0) {
    set_err("unexpected VMM granularity " + std::to_string(gran));
    return CDPROBE_ERR_UNSUPPORTED;
  }
  r = create_alloc(h, L.ordinal, ht, m.bytes, &m.own[li]);
  if (r != CUDA_SUCCESS) return fail_drv(h, "cuMemCreate", r);
  m.has_own[li] = true;
  if (h->handle_type == 1u) {
    int fd = -1;
    r = h->drv.MemExportToShareableHandle(&fd, m.own[li], CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
    if (r != CUDA_SUCCESS) return fail_drv(h, "cuMemExportToShareableHandle(fd)", r);
    m.own_fd[li] = fd;
  }
  return CDPROBE_OK;
}

// What each process reports at a step of a collective setup: its return code and message and, where the step hands
// something over, a payload (ensure_nvls: the area's size and the multicast object's fabric handle).
struct StepReport {
  int32_t rc;
  char msg[124];
  uint64_t bytes;
  CUmemFabricHandle fabric;
};

// Every process's rc, shared: the first failure in process order wins, with its message, so that no process goes on
// to an exchange another has left.  A failed exchange is CDPROBE_ERR_RENDEZVOUS.  `mine_in` (optional) is this
// process's payload, and `first` (optional) gets the report of the process hosting rank 0.
static int agree_step(cdprobe* h, int rc, const StepReport* mine_in = nullptr, StepReport* first = nullptr) {
  StepReport mine;
  memset(&mine, 0, sizeof(mine));
  if (mine_in != nullptr) mine = *mine_in;
  mine.rc = rc;
  if (rc != CDPROBE_OK) snprintf(mine.msg, sizeof(mine.msg), "%s", g_last_error.c_str());
  std::vector<StepReport> all(h->cfg.world_size, mine);
  if (h->cfg.world_size > 1) {
    std::string err;
    if (h->rdv.allgather(&mine, sizeof(mine), all.data(), &err) != 0) {
      set_err(err);
      return CDPROBE_ERR_RENDEZVOUS;
    }
  }
  if (first != nullptr) *first = all[0];
  for (uint32_t p = 0; p < all.size(); ++p)
    if (all[p].rc != CDPROBE_OK) {
      if (p != h->cfg.rank) set_err(all[p].msg);  // this process's own message stays whole
      return all[p].rc;
    }
  return CDPROBE_OK;
}

// Creates m with allocations of `bytes`: one per local rank, exported and exchanged with every process over the
// rendezvous, the other processes' imported, and rank j's mapped into local rank li wherever st[its rank][j] is 0 on
// entry.  st[its rank][j] then holds the outcome: the import's CUresult, CDPROBE_ERR_UNSUPPORTED between MIG
// instances, or map_peer's status.  With `agree`, the processes first share whether each created its allocations
// (agree_step); without it (open, whose failure ends the handle), a failure returns at once.  On failure the caller
// releases m.
static int share_alloc(cdprobe* h, SharedAlloc& m, size_t bytes, int32_t (*st)[kMaxRanks], bool agree) {
  const cdprobe_config_t& c = h->cfg;
  std::string err;
  m.bytes = bytes;
  int rc = CDPROBE_OK;
  for (uint32_t li = 0; li < h->n_local && rc == CDPROBE_OK; ++li) rc = create_own(h, m, li);
  if (agree) rc = agree_step(h, rc);
  if (rc != CDPROBE_OK) return rc;

  // ---- exchange handles between processes ---------------------------------
  if (c.world_size > 1) {
    if (h->handle_type == 1u) {
      int mine[kMaxRanks];
      for (uint32_t li = 0; li < h->n_local; ++li) mine[li] = m.own_fd[li];
      std::vector<int> all;
      if (h->rdv.allgather_fds(mine, h->n_local, &all, &err) != 0) {
        set_err(err);
        return CDPROBE_ERR_RENDEZVOUS;
      }
      for (uint32_t j = 0; j < h->n_total; ++j) {
        const bool local = j >= h->first && j < h->first + h->n_local;
        if (!local) {
          CUresult r = h->drv.MemImportFromShareableHandle(&m.imported[j], (void*)(uintptr_t)all[j],
                                                           CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
          if (r == CUDA_SUCCESS) m.has_import[j] = true;
          else
            for (uint32_t li = 0; li < h->n_local; ++li) st[h->first + li][j] = (int32_t)r;
        }
        ::close(all[j]);
      }
    } else {
      CUmemFabricHandle mine[kMaxRanks], all[kMaxRanks];
      memset(mine, 0, sizeof(mine));
      for (uint32_t li = 0; li < h->n_local; ++li) {
        CUresult r = h->drv.MemExportToShareableHandle(&mine[li], m.own[li], CU_MEM_HANDLE_TYPE_FABRIC, 0);
        if (r != CUDA_SUCCESS) return fail_drv(h, "cuMemExportToShareableHandle(fabric)", r);
      }
      if (h->rdv.allgather(mine, sizeof(CUmemFabricHandle) * h->n_local, all, &err) != 0) {
        set_err(err);
        return CDPROBE_ERR_RENDEZVOUS;
      }
      for (uint32_t j = 0; j < h->n_total; ++j) {
        const bool local = j >= h->first && j < h->first + h->n_local;
        if (local) continue;
        CUresult r = h->drv.MemImportFromShareableHandle(&m.imported[j], &all[j], CU_MEM_HANDLE_TYPE_FABRIC);
        if (r == CUDA_SUCCESS) m.has_import[j] = true;
        else
          for (uint32_t li = 0; li < h->n_local; ++li) st[h->first + li][j] = (int32_t)r;
      }
    }
  }

  // ---- map every rank's allocation into every local rank's address space --
  for (uint32_t li = 0; li < h->n_local; ++li) {
    LocalRank& L = h->lr[li];
    for (uint32_t j = 0; j < h->n_total; ++j) {
      int32_t s = st[L.grank][j];
      if (s == 0) {
        if (j != L.grank && L.mig && (c.flags & (CDPROBE_FLAG_MIG_AWARE | CDPROBE_FLAG_SIMULATE_MIG)))
          s = CDPROBE_ERR_UNSUPPORTED;  // no P2P under MIG (SURVEY H8): identity matrix, "not applicable"
        else s = map_peer(h, m, li, j);
      }
      st[L.grank][j] = s;
    }
  }
  return CDPROBE_OK;
}

// Every process's rows of a mapping-status matrix (local ranks' rows filled in), gathered into every row of st.
static int gather_status(cdprobe* h, int32_t (*st)[kMaxRanks]) {
  if (h->cfg.world_size == 1) return CDPROBE_OK;
  std::string err;
  int32_t mine[kMaxRanks][kMaxRanks], all[kMaxRanks][kMaxRanks][kMaxRanks];
  memset(mine, 0, sizeof(mine));
  for (uint32_t li = 0; li < h->n_local; ++li) memcpy(mine[li], st[h->first + li], sizeof(mine[li]));
  if (h->rdv.allgather(mine, sizeof(int32_t) * kMaxRanks * h->n_local, all, &err) != 0) {
    set_err(err);
    return CDPROBE_ERR_RENDEZVOUS;
  }
  const int32_t* flat = &all[0][0][0];
  for (uint32_t g = 0; g < h->n_total; ++g) memcpy(st[g], flat + (size_t)g * kMaxRanks, sizeof(st[g]));
  return CDPROBE_OK;
}

// Returns a collective setup's rc.  On failure, first releases what the setup made, keeping its message in
// cdprobe_last_error, so that nothing is kept and the next call tries again.
template <class Release>
static int release_on_failure(int rc, Release release) {
  if (rc != CDPROBE_OK) {
    const std::string keep = g_last_error;
    release();
    g_last_error = keep;
  }
  return rc;
}

int ensure_area(cdprobe* h, SharedAlloc& m, size_t bytes) {
  if (m.bytes != 0) return CDPROBE_OK;
  bytes = (bytes + kVmmGranule - 1) / kVmmGranule * kVmmGranule;
  int32_t st[kMaxRanks][kMaxRanks] = {};
  for (uint32_t li = 0; li < h->n_local; ++li)
    for (uint32_t j = 0; j < h->n_total; ++j) st[h->lr[li].grank][j] = cell_status(h, li, j);
  int rc = share_alloc(h, m, bytes, st, true);
  if (rc == CDPROBE_OK) rc = gather_status(h, st);
  if (rc == CDPROBE_OK) memcpy(m.status, st, sizeof(st));
  return release_on_failure(rc, [&] { release_shared(h, m); });
}

// Unmaps the NVLS area in every local rank, unbinds every local device from the multicast object, then releases the
// object and the allocations: no binding outlives its mapping, and no object its bindings.
static void release_nvls(cdprobe* h) {
  NvlsArea& a = h->nvls;
  for (uint32_t li = 0; li < h->n_local; ++li) {
    if (h->lr[li].ordinal < 0) continue;
    cudaSetDevice(h->lr[li].ordinal);
    if (a.mc_mapped[li]) unmap_range(h, a.mc_va[li], a.bytes);
    if (a.uc_mapped[li]) unmap_range(h, a.uc_va[li], a.bytes);
  }
  for (uint32_t li = 0; li < h->n_local; ++li) {
    CUdevice dev;
    if (a.bound[li] && h->drv.DeviceGet(&dev, h->lr[li].ordinal) == CUDA_SUCCESS)
      h->drv.MulticastUnbind(a.mc, dev, 0, a.bytes);
  }
  if (a.has_mc) h->drv.MemRelease(a.mc);
  for (uint32_t li = 0; li < h->n_local; ++li) {
    if (!a.has_own[li]) continue;
    cudaSetDevice(h->lr[li].ordinal);
    h->drv.MemRelease(a.own[li]);
  }
  a = NvlsArea();
}

static int ensure_nvls_steps(cdprobe* h, size_t bytes, bool* refused) {
  NvlsArea& a = h->nvls;
  // a multicast object needs a shareable handle type even in one process (cuMulticastCreate refuses none)
  const CUmemAllocationHandleType ht =
      h->handle_type == 8u ? CU_MEM_HANDLE_TYPE_FABRIC : CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  const bool host0 = h->first == 0;
  CUmulticastObjectProp mp;
  memset(&mp, 0, sizeof(mp));
  mp.numDevices = h->n_total;
  mp.handleTypes = ht;
  // 1. the size, and in the process hosting rank 0 the object, exported for the others
  StepReport mine;
  memset(&mine, 0, sizeof(mine));
  int fd = -1;
  int rc = CDPROBE_OK;
  size_t gran = 0;
  mp.size = bytes;
  CUresult r = h->drv.MulticastGetGranularity(&gran, &mp, CU_MULTICAST_GRANULARITY_MINIMUM);
  if (r != CUDA_SUCCESS) rc = fail_drv(h, "cuMulticastGetGranularity", r);
  if (rc == CDPROBE_OK && (gran == 0 || gran % kVmmGranule != 0 && kVmmGranule % gran != 0)) {
    set_err("unexpected multicast granularity " + std::to_string(gran));
    rc = CDPROBE_ERR_UNSUPPORTED;
  }
  const size_t align = std::max<size_t>(gran, kVmmGranule);
  mp.size = mine.bytes = (bytes + align - 1) / align * align;
  if (rc == CDPROBE_OK && host0) {
    r = h->drv.MulticastCreate(&a.mc, &mp);
    if (r != CUDA_SUCCESS) rc = fail_drv(h, "cuMulticastCreate", r);
    else a.has_mc = true;
    *refused = h->n_total == 1 && r == CUDA_ERROR_INVALID_VALUE;
    if (*refused) set_err(g_last_error + " (the driver refuses a multicast object of one device)");
    if (rc == CDPROBE_OK && h->cfg.world_size > 1 && ht == CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR) {
      r = h->drv.MemExportToShareableHandle(&fd, a.mc, ht, 0);
      if (r != CUDA_SUCCESS) rc = fail_drv(h, "cuMemExportToShareableHandle(multicast fd)", r);
    } else if (rc == CDPROBE_OK && h->cfg.world_size > 1 && ht == CU_MEM_HANDLE_TYPE_FABRIC) {
      r = h->drv.MemExportToShareableHandle(&mine.fabric, a.mc, ht, 0);
      if (r != CUDA_SUCCESS) rc = fail_drv(h, "cuMemExportToShareableHandle(multicast fabric)", r);
    }
  }
  StepReport host0_report;
  rc = agree_step(h, rc, &mine, &host0_report);
  if (rc != CDPROBE_OK) {
    if (fd >= 0) ::close(fd);
    return rc;
  }
  a.bytes = host0_report.bytes;
  // 2. the handle to the other processes.  allgather_fds takes one descriptor from every process: the others send
  //    their probe allocation's, which every receiver closes unread
  if (h->cfg.world_size > 1 && ht == CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR) {
    std::vector<int> all;
    std::string err;
    const int send = host0 ? fd : h->mem.own_fd[0];
    const int xrc = h->rdv.allgather_fds(&send, 1, &all, &err);
    if (fd >= 0) ::close(fd);
    if (xrc != 0) {
      set_err(err);
      return CDPROBE_ERR_RENDEZVOUS;
    }
    if (!host0) {
      r = h->drv.MemImportFromShareableHandle(&a.mc, (void*)(uintptr_t)all[0], ht);
      if (r != CUDA_SUCCESS) rc = fail_drv(h, "cuMemImportFromShareableHandle(multicast fd)", r);
      else a.has_mc = true;
    }
    for (int f : all) ::close(f);
  } else if (h->cfg.world_size > 1 && !host0) {
    r = h->drv.MemImportFromShareableHandle(&a.mc, &host0_report.fabric, ht);
    if (r != CUDA_SUCCESS) rc = fail_drv(h, "cuMemImportFromShareableHandle(multicast fabric)", r);
    else a.has_mc = true;
  }
  // 3. every process adds its devices; binding or mapping blocks until every device is added, so nobody starts
  //    before every process has reported that it did
  for (uint32_t li = 0; li < h->n_local && rc == CDPROBE_OK; ++li) {
    CUdevice dev;
    r = h->drv.DeviceGet(&dev, h->lr[li].ordinal);
    if (r == CUDA_SUCCESS) r = h->drv.MulticastAddDevice(a.mc, dev);
    if (r != CUDA_SUCCESS) rc = fail_drv(h, "cuMulticastAddDevice", r);
  }
  if ((rc = agree_step(h, rc)) != CDPROBE_OK) return rc;
  // 4. per local rank: its allocation, bound at offset 0, then the object and the allocation mapped into it
  for (uint32_t li = 0; li < h->n_local && rc == CDPROBE_OK; ++li) {
    LocalRank& L = h->lr[li];
    if (cudaSetDevice(L.ordinal) != cudaSuccess) {
      set_err("cudaSetDevice");
      rc = CDPROBE_ERR_CUDA;
      break;
    }
    r = create_alloc(h, L.ordinal, ht, a.bytes, &a.own[li]);
    if (r != CUDA_SUCCESS) {
      rc = fail_drv(h, "cuMemCreate", r);
      break;
    }
    a.has_own[li] = true;
    r = h->drv.MulticastBindMem(a.mc, 0, a.own[li], 0, a.bytes, 0);
    if (r != CUDA_SUCCESS) {
      rc = fail_drv(h, "cuMulticastBindMem", r);
      break;
    }
    a.bound[li] = true;
    r = map_range(h, a.mc, a.bytes, align, L.ordinal, &a.mc_va[li]);
    if (r != CUDA_SUCCESS) {
      rc = fail_drv(h, "cuMemMap(multicast)", r);
      break;
    }
    a.mc_mapped[li] = true;
    r = map_range(h, a.own[li], a.bytes, align, L.ordinal, &a.uc_va[li]);
    if (r != CUDA_SUCCESS) {
      rc = fail_drv(h, "cuMemMap(unicast)", r);
      break;
    }
    a.uc_mapped[li] = true;
  }
  return agree_step(h, rc);
}

int ensure_nvls(cdprobe* h, size_t bytes, bool* refused) {
  *refused = false;
  if (h->nvls.bytes != 0) return CDPROBE_OK;
  return release_on_failure(ensure_nvls_steps(h, bytes, refused), [h] { release_nvls(h); });
}

// Phase table of local rank li: see schedule.cc.
static int build_phases(cdprobe* h, uint32_t li) {
  LocalRank& L = h->lr[li];
  ScheduleInput in;
  in.plan = &h->plan;
  in.rank = L.grank;
  in.ops = h->cfg.ops;
  in.flags = h->cfg.flags;
  in.ctas = L.ctas;
  in.verify_ctas = h->verify_ctas;
  in.status = h->status;
  const int rc = make_phases(in, L.phases, &L.n_phases, &L.peer_mask);
  if (rc != CDPROBE_OK) set_err("schedule needs more than CDPROBE_MAX_PHASES phases (use overlap-verify or fewer ops)");
  return rc;
}

static int rebuild_all(cdprobe* h) {
  for (uint32_t li = 0; li < h->n_local; ++li) {
    const int rc = build_phases(h, li);
    if (rc != CDPROBE_OK) return rc;
  }
  return CDPROBE_OK;
}

// Sets or clears one schedule flag and rebuilds every phase table; on failure the old flags and tables come back.
static int set_flag(cdprobe* h, uint32_t flag, bool on) {
  const uint32_t old = h->cfg.flags;
  h->cfg.flags = (old & ~flag) | (on ? flag : 0u);
  const int rc = rebuild_all(h);
  if (rc != CDPROBE_OK) {
    h->cfg.flags = old;
    rebuild_all(h);
  }
  return rc;
}

// The option that arms each measurement's test fault (cdprobe_set_option).  Every value is accepted when it is set:
// what it names depends on the domain and the call's arguments, so the call checks it.
struct FaultOption {
  uint32_t option;
  Measurement meas;
};
constexpr FaultOption kFaultOptions[] = {
    {CDPROBE_OPT_PINGPONG_FAULT, kMeasPingPong},
    {CDPROBE_OPT_ATOMICS_FAULT, kMeasAtomics},
    {CDPROBE_OPT_ALLREDUCE_FAULT, kMeasAllReduce},
    {CDPROBE_OPT_ALLTOALL_FAULT, kMeasAllToAll},
    {CDPROBE_OPT_ALLREDUCE_TWOSHOT_FAULT, kMeasTwoShot},
    {CDPROBE_OPT_ALLREDUCE_LL_FAULT, kMeasLl},
    {CDPROBE_OPT_ALLREDUCE_RING_FAULT, kMeasRing},
    {CDPROBE_OPT_ALLREDUCE_PUSH_FAULT, kMeasPush},
    {CDPROBE_OPT_ALLREDUCE_NVLS_FAULT, kMeasNvls},
    {CDPROBE_OPT_MEMCPY_FAULT, kMeasMemcpy},
    {CDPROBE_OPT_CE_ALLTOALL_FAULT, kMeasCeAllToAll},
};

static void fill_params(const cdprobe* h, uint32_t li, const Phase* phases, uint32_t n_phases, uint32_t peer_mask,
                        ProbeParams* P) {
  const LocalRank& L = h->lr[li];
  memset(P, 0, sizeof(*P));
  for (uint32_t j = 0; j < h->n_total; ++j)
    P->base_peer[j] = h->mem.mapped[li][j] ? reinterpret_cast<uint8_t*>(h->mem.va[li][j]) : nullptr;
  P->row = L.row;
  P->run_seq = h->launch_seq;
  P->seq_base = h->launch_seq * (uint64_t)(kMaxPhases + 2);
  P->timeout_ns = timeout_ns(h);
  P->bpp = h->plan.bpp;
  P->src_off = h->plan.src_off;
  P->land_off = h->plan.land_off;
  P->rank = L.grank;
  P->n_ranks = h->n_total;
  P->n_phases = n_phases;
  P->peer_mask = peer_mask;
  P->path = h->path;
  P->full_mode = h->plan.full ? 1u : 0u;
  for (uint32_t p = 0; p < n_phases; ++p) {
    P->phase[p] = phases[p];
    for (int jb = 0; jb < 2; ++jb) {
      Job& job = P->phase[p].job[jb];
      if (job.kind == kJobWrite) job.salt = write_salt(h->seed, L.grank, (uint32_t)job.peer, h->launch_seq);
      if (job.kind == kJobWarm) job.salt = h->warm_now ? h->warm_bytes : 0ull;
    }
  }
}

// Waits until every local row carries `token`; returns false on host timeout or a kernel error.
// The rows are pinned host words the kernels write themselves.  A healthy probe is over in 0.5-3.3 ms,
// so the wait spins hot for as long as a healthy run can plausibly take (twice the previous run, at
// least 2 ms, at most 50 ms) and then backs off to a 100 us sleep between polls: a hung peer costs the
// daemon pod a sleeping thread for timeout_ms, not a core burnt inside its CPU limit.
static bool wait_rows(cdprobe* h, uint64_t token) {
  const double t_begin = now_ms();
  const double t_end = t_begin + h->cfg.timeout_ms + 2000.0;
  double hot_ms = 2.0 * h->last_probe_ms;
  if (hot_ms < 2.0) hot_ms = 2.0;
  if (hot_ms > 50.0) hot_ms = 50.0;
  const double t_hot = t_begin + hot_ms;
  bool hot = true;
  uint32_t spins = 0;
  for (;;) {
    bool all = true;
    for (uint32_t li = 0; li < h->n_local; ++li) {
      if (h->lr[li].row->done != token) {
        all = false;
        break;
      }
    }
    if (all) {
      __sync_synchronize();
      return true;
    }
    if (!hot) {
      timespec ts = {0, 100000};
      nanosleep(&ts, nullptr);
    }
    if (!hot || (++spins & 0x3ffu) == 0) {
      const double t = now_ms();
      if (t > t_end) return false;
      if (hot && t > t_hot) hot = false;
      if (hot || (++spins & 0x3fu) == 0) {
        // surface asynchronous launch/kernel errors instead of waiting on them
        for (uint32_t li = 0; li < h->n_local; ++li) {
          if (h->solo_rank && h->solo_rank != li + 1) continue;
          cudaSetDevice(h->lr[li].ordinal);
          cudaError_t q = cudaStreamQuery(h->lr[li].stream);
          if (q != cudaSuccess && q != cudaErrorNotReady) {
            set_err(std::string("kernel failed: ") + cudaGetErrorName(q));
            return false;
          }
        }
      }
    }
  }
}

static int reset_ctrl_local(cdprobe* h, uint32_t li) {
  LocalRank& L = h->lr[li];
  CDP_RT(cudaSetDevice(L.ordinal));
  uint8_t* base = reinterpret_cast<uint8_t*>(h->mem.va[li][L.grank]);
  const size_t off = offsetof(Ctrl, grid_arrive);
  CDP_RT(cudaMemsetAsync(base + off, 0, sizeof(Ctrl) - off, L.stream));
  CDP_RT(cudaStreamSynchronize(L.stream));
  return CDPROBE_OK;
}

// Writes local rank li's landing-fault descriptor (cdprobe_corrupt_landing), stream-ordered after the last run.
static int write_fault(cdprobe* h, uint32_t li, const LandingFault& f) {
  LocalRank& L = h->lr[li];
  CDP_RT(cudaSetDevice(L.ordinal));
  uint8_t* p = reinterpret_cast<uint8_t*>(h->mem.va[li][L.grank]) + offsetof(Ctrl, fault);
  CDP_RT(cudaMemcpyAsync(p, &f, sizeof(f), cudaMemcpyHostToDevice, L.stream));
  CDP_RT(cudaStreamSynchronize(L.stream));
  return CDPROBE_OK;
}

static int launch_one(cdprobe* h, uint32_t li, const ProbeParams& P) {
  LocalRank& L = h->lr[li];
  CDP_RT(cudaSetDevice(L.ordinal));
  cudaError_t e = (cudaError_t)probe_kernel_launch(&P, L.ctas, launch_cooperatively(h, L), L.stream);
  if (e != cudaSuccess) return fail_cuda("launch cdprobe_kernel", e);
  return CDPROBE_OK;
}

// Open-time: fill the source pattern and let the probe kernel itself compute the
// slice checksums that readers will compare against (published in Ctrl).
static int fill_and_publish(cdprobe* h) {
  const Plan& pl = h->plan;
  h->launch_seq++;
  for (uint32_t li = 0; li < h->n_local; ++li) {
    LocalRank& L = h->lr[li];
    CDP_RT(cudaSetDevice(L.ordinal));
    uint8_t* base = reinterpret_cast<uint8_t*>(h->mem.va[li][L.grank]);
    CDP_RT(cudaMemsetAsync(base, 0, kCtrlBytes, L.stream));
    CDP_RT(cudaMemsetAsync(base + pl.land_off, 0, pl.land_bytes, L.stream));
    cudaError_t e = (cudaError_t)probe_fill_launch(base + pl.src_off, pl.src_bytes, h->seed, L.grank,
                                                   (unsigned)L.sm_count * 8u, L.stream);
    if (e != cudaSuccess) return fail_cuda("launch fill kernel", e);
    Phase ph[kMaxPhases];
    memset(ph, 0, sizeof(ph));
    for (uint32_t s = 0; s < pl.n_slices; ++s) {
      ph[s].job[0].kind = kJobRead;
      ph[s].job[0].peer = (int8_t)L.grank;
      ph[s].job[0].slot = (uint8_t)s;
      ph[s].job[0].cta0 = 0;
      ph[s].job[0].nctas = (uint16_t)L.ctas;
      ph[s].sync_mask = 0;
      ph[s].post_mask = 0;
    }
    ProbeParams P;
    fill_params(h, li, ph, pl.n_slices, 0u, &P);
    L.row->done = 0;
    const int rc = launch_one(h, li, P);
    if (rc != CDPROBE_OK) return rc;
  }
  if (!wait_rows(h, h->launch_seq)) {
    h->sticky = true;
    if (g_last_error.empty()) set_err("timeout computing source checksums");
    return CDPROBE_ERR_TIMEOUT;
  }
  for (uint32_t li = 0; li < h->n_local; ++li) {
    LocalRank& L = h->lr[li];
    CDP_RT(cudaSetDevice(L.ordinal));
    if (L.row->aborted) {
      set_err("device watchdog fired while computing source checksums");
      return CDPROBE_ERR_TIMEOUT;
    }
    uint64_t pub[2][kMaxRanks];
    memset(pub, 0, sizeof(pub));
    for (uint32_t s = 0; s < pl.n_slices; ++s) {
      pub[0][s] = h->src_sum[li][s] = L.row->ph[s].sum[0];
      pub[1][s] = h->src_xor[li][s] = L.row->ph[s].xr[0];
    }
    uint8_t* base = reinterpret_cast<uint8_t*>(h->mem.va[li][L.grank]);
    CDP_RT(cudaMemcpyAsync(base + offsetof(Ctrl, src_sum), pub[0], sizeof(pub[0]), cudaMemcpyHostToDevice, L.stream));
    CDP_RT(cudaMemcpyAsync(base + offsetof(Ctrl, src_xor), pub[1], sizeof(pub[1]), cudaMemcpyHostToDevice, L.stream));
    CDP_RT(cudaStreamSynchronize(L.stream));
  }
  return CDPROBE_OK;
}

static void destroy(cdprobe* h) {
  if (h == nullptr) return;
  for (uint32_t li = 0; li < h->n_local; ++li) {
    LocalRank& L = h->lr[li];
    if (L.ordinal < 0) continue;
    cudaSetDevice(L.ordinal);
    if (L.stream) cudaStreamSynchronize(L.stream);
  }
  release_nvls(h);
  release_shared(h, h->push);
  release_shared(h, h->ring);
  release_shared(h, h->ll);
  release_shared(h, h->gather);
  release_shared(h, h->area);
  release_shared(h, h->mem);
  for (uint32_t li = 0; li < h->n_local; ++li) {
    LocalRank& L = h->lr[li];
    if (L.ordinal < 0) continue;
    cudaSetDevice(L.ordinal);
    if (L.row) cudaFreeHost(L.row);
    if (L.scratch) cudaFree(L.scratch);
    if (L.ev0) cudaEventDestroy(L.ev0);
    if (L.ev1) cudaEventDestroy(L.ev1);
    for (uint32_t i = 0; i < (uint32_t)kMaxRanks; ++i) {
      if (L.cea_stream[i]) cudaStreamSynchronize(L.cea_stream[i]);
      for (cudaEvent_t ev : L.cea_copy_ev[i])
        if (ev) cudaEventDestroy(ev);
      if (L.cea_stream[i]) cudaStreamDestroy(L.cea_stream[i]);
    }
    for (cudaEvent_t ev : L.rep_ev)
      if (ev) cudaEventDestroy(ev);
    if (L.stream) cudaStreamDestroy(L.stream);
  }
  if (h->copy_host) cudaFreeHost(h->copy_host);
  delete h->links;
  h->rdv.close();
  delete h;
}

static int open_impl(const cdprobe_config_t* cfg, cdprobe* h) {
  const double t0 = now_ms();
  h->cfg = *cfg;
  cdprobe_config_t& c = h->cfg;
  if (c.ops == 0) c.ops = CDPROBE_OP_READ | CDPROBE_OP_WRITE;
  if (c.ops & ~(CDPROBE_OP_READ | CDPROBE_OP_WRITE)) return CDPROBE_ERR_ARG;
  if (c.timeout_ms == 0) c.timeout_ms = 5000;
  // gate: see gate_gbps(); 0 in either field selects the default at verdict time
  if (c.link_peak_gbps < 0.f || c.min_fraction < 0.f) return CDPROBE_ERR_ARG;
  if (c.world_size == 0) c.world_size = 1;
  if (c.rank >= c.world_size) return CDPROBE_ERR_ARG;
  h->path = (c.flags & CDPROBE_FLAG_PATH_LDST) ? 1u : 0u;
  if (!(c.flags & CDPROBE_FLAG_SERIAL_VERIFY)) c.flags |= CDPROBE_FLAG_OVERLAP_VERIFY;  // overlapped verify is the default
  h->seed = c.seed ? c.seed : kDefaultSeed;
  // the hardware queues per device the CUDA runtime of this process gives its streams (cdprobe_ce_alltoall); it reads
  // the variable once, at its initialisation, and clamps it to [1, 32]
  if (const char* mc = getenv("CUDA_DEVICE_MAX_CONNECTIONS"); mc != nullptr && *mc != '\0') {
    const long v = strtol(mc, nullptr, 10);
    if (v > 0) h->max_connections = (uint32_t)std::min(v, 32L);
  }
  c.session[sizeof(c.session) - 1] = '\0';
  memset(h->status, 0, sizeof(h->status));

  std::string err;
  cudaError_t e = h->drv.load(&err);
  if (e != cudaSuccess) {
    set_err(err);
    return CDPROBE_ERR_NO_DEVICE;
  }
  int ndev = 0;
  e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess) return fail_cuda("cudaGetDeviceCount", e);
  if (ndev <= 0) {
    set_err("no CUDA device visible");
    return CDPROBE_ERR_NO_DEVICE;
  }
  if (c.n_gpus == 0) {
    c.n_gpus = ndev > kMaxRanks ? kMaxRanks : (uint32_t)ndev;
    for (uint32_t i = 0; i < c.n_gpus; ++i) c.ordinals[i] = (int32_t)i;
  }
  if (c.n_gpus > (uint32_t)kMaxRanks) return CDPROBE_ERR_ARG;
  for (uint32_t i = 0; i < c.n_gpus; ++i) {
    if (c.ordinals[i] < 0 || c.ordinals[i] >= ndev) {
      set_err("ordinal out of range");
      return CDPROBE_ERR_ARG;
    }
    if (!(c.flags & CDPROBE_FLAG_ALLOW_SAME_DEVICE))
      for (uint32_t k = 0; k < i; ++k)
        if (c.ordinals[k] == c.ordinals[i]) {
          set_err("duplicate ordinal (set CDPROBE_FLAG_ALLOW_SAME_DEVICE for tests)");
          return CDPROBE_ERR_ARG;
        }
  }
  h->n_local = c.n_gpus;
  h->n_total = c.n_gpus * c.world_size;
  h->first = c.rank * c.n_gpus;
  if (h->n_total > (uint32_t)kMaxRanks) {
    set_err("more than CDPROBE_MAX_GPUS ranks");
    return CDPROBE_ERR_ARG;
  }
  int rc = make_plan(h->n_total, c.bytes, c.mode, c.flags, &h->plan);
  if (rc != CDPROBE_OK) {
    set_err("invalid bytes/mode for this domain size");
    return rc;
  }

  if (c.world_size > 1) {
    if (h->rdv.connect(c.session, c.rank, c.world_size, c.timeout_ms + 20000, &err) != 0) {
      set_err(err);
      return CDPROBE_ERR_RENDEZVOUS;
    }
    uint32_t mine = c.n_gpus, all[kMaxRanks * 4];
    if (c.world_size > (uint32_t)kMaxRanks || h->rdv.allgather(&mine, sizeof(mine), all, &err) != 0) {
      set_err(err);
      return CDPROBE_ERR_RENDEZVOUS;
    }
    for (uint32_t r = 0; r < c.world_size; ++r)
      if (all[r] != c.n_gpus) {
        set_err("every process must drive the same number of GPUs");
        return CDPROBE_ERR_ARG;
      }
  }

  const bool want_fabric = (c.flags & CDPROBE_FLAG_FABRIC_HANDLES) && imex_channel0_present();
  h->handle_type = want_fabric ? 8u : (c.world_size > 1 ? 1u : 0u);
  if (c.world_size > 1 && h->rdv.is_tcp() && !want_fabric) {
    set_err("a tcp: rendezvous spans nodes: it needs CDPROBE_FLAG_FABRIC_HANDLES and /dev/nvidia-caps-imex-channels/channel0");
    return CDPROBE_ERR_UNSUPPORTED;
  }

  // ---- per local rank: device, stream, allocation, result row -------------
  for (uint32_t li = 0; li < h->n_local; ++li) {
    LocalRank& L = h->lr[li];
    L.grank = h->first + li;
    L.ordinal = c.ordinals[li];
    CDP_RT(cudaSetDevice(L.ordinal));
    CDP_RT(cudaFree(0));
    cudaDeviceProp prop;
    CDP_RT(cudaGetDeviceProperties(&prop, L.ordinal));
    if (prop.major != 9 || prop.minor != 0) {
      set_err(std::string("device is sm_") + std::to_string(prop.major * 10 + prop.minor) +
              "; libcdprobe carries sm_90a code only");
      return CDPROBE_ERR_UNSUPPORTED;
    }
    L.sm_count = prop.multiProcessorCount;
    L.mig = strstr(prop.name, "MIG") != nullptr || (c.flags & CDPROBE_FLAG_SIMULATE_MIG);
    format_uuid(prop.uuid, L.mig, L.uuid);
    int coop = 0;
    CDP_RT(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, L.ordinal));
    L.coop = coop != 0;
    int per_sm = 0;
    e = (cudaError_t)probe_kernel_prepare(&per_sm);
    if (e != cudaSuccess) return fail_cuda("prepare cdprobe_kernel", e);
    if (per_sm < 1) {
      set_err("persistent kernel does not fit an SM");
      return CDPROBE_ERR_UNSUPPORTED;
    }
    uint32_t ctas = c.ctas ? c.ctas : (uint32_t)L.sm_count;
    const uint32_t cap = (uint32_t)L.sm_count * (uint32_t)per_sm;
    if (ctas > cap) ctas = cap;
    if (ctas > 65535u) ctas = 65535u;
    L.ctas = ctas;
    L.max_ctas = (int)(cap > 65535u ? 65535u : cap);
    CDP_RT(cudaStreamCreateWithFlags(&L.stream, cudaStreamNonBlocking));
    CDP_RT(cudaEventCreate(&L.ev0));
    CDP_RT(cudaEventCreate(&L.ev1));

    void* row = nullptr;
    CDP_RT(cudaHostAlloc(&row, sizeof(ResultRow), cudaHostAllocPortable | cudaHostAllocMapped));
    memset(row, 0, sizeof(ResultRow));
    L.row = static_cast<ResultRow*>(row);
  }

  // ---- every rank's device, by UUID: which cells of a run cross a device boundary (cdprobe_links) ----
  for (uint32_t li = 0; li < h->n_local; ++li) memcpy(h->rank_uuid[h->first + li], h->lr[li].uuid, 48);
  if (c.world_size > 1) {
    std::vector<char> all((size_t)c.world_size * c.n_gpus * 48);
    if (h->rdv.allgather(h->rank_uuid[h->first], (size_t)c.n_gpus * 48, all.data(), &err) != 0) {
      set_err(err);
      return CDPROBE_ERR_RENDEZVOUS;
    }
    memcpy(h->rank_uuid, all.data(), all.size());
  }

  // ---- the probe allocations, shared with every process and mapped ---------
  rc = share_alloc(h, h->mem, h->plan.alloc_bytes, h->status, false);
  if (rc != CDPROBE_OK) return rc;
  for (uint32_t li = 0; li < h->n_local; ++li) {
    const LocalRank& L = h->lr[li];
    if (h->status[L.grank][L.grank] != 0) {
      set_err("cannot map own allocation: " + h->drv.error_name((CUresult)h->status[L.grank][L.grank]));
      return CDPROBE_ERR_CUDA;
    }
  }
  rc = gather_status(h, h->status);
  if (rc != CDPROBE_OK) return rc;
  rc = rebuild_all(h);
  if (rc != CDPROBE_OK) return rc;
  h->open_ms = now_ms() - t0;

  const double t1 = now_ms();
  rc = fill_and_publish(h);
  if (rc != CDPROBE_OK) return rc;
  h->fill_ms = now_ms() - t1;
  // nobody may start probing before every rank has published its checksums
  if (c.world_size > 1 && h->rdv.barrier(&err) != 0) {
    set_err(err);
    return CDPROBE_ERR_RENDEZVOUS;
  }
  return CDPROBE_OK;
}

// The GB/s an ordered pair must reach for a passing verdict (0: bandwidth is not judged).
//   link_peak_gbps > 0 : absolute, min_fraction x link_peak_gbps (default fraction 0.65: the round-1 gate
//                        against nominal 900).
//   link_peak_gbps == 0: the nominal NVLink 4 rate of an H100 SXM (450 GB/s per direction, data sheet) for every
//                        op and schedule, de-rated for the fixed cost of a phase (ramp and drain: 6 us, the
//                        fixed cost of a read phase measured on an H100 at N = 1); default fraction 0.65.  What
//                        healthy H100 NVLink delivers to SM-issued traffic has not been measured, so the default
//                        fraction leaves a wide margin below nominal; set link_peak_gbps / min_fraction to gate
//                        tighter once a domain's healthy rate is known.
constexpr double kNominalLinkGbps = 450.0;
constexpr double kPhaseOverheadNs = 6000.0;
static float gate_gbps_for(const cdprobe_config_t& cfg, uint32_t n_total, uint64_t bpp, bool is_read) {
  (void)is_read;
  if (cfg.mode == CDPROBE_MODE_REACH_ONLY || n_total <= 1) return 0.f;
  const float fraction = cfg.min_fraction > 0.f ? cfg.min_fraction : 0.65f;
  if (cfg.link_peak_gbps > 0.f) return fraction * cfg.link_peak_gbps;
  const double b = (double)bpp;
  const double expected = b / (b / kNominalLinkGbps + kPhaseOverheadNs);  // bytes per ns == GB/s
  return (float)(fraction * expected);
}
static float gate_gbps(const cdprobe* h, bool is_read) { return gate_gbps_for(h->cfg, h->n_total, h->plan.bpp, is_read); }

static void assemble(const cdprobe* h, cdprobe_result_t* out) {
  const Plan& pl = h->plan;
  const float gate_r = gate_gbps(h, true), gate_w = gate_gbps(h, false);
  out->gate_gbps_read = gate_r;
  out->gate_gbps_write = gate_w;
  bool verdict = true;
  float min_r = 0.f, min_w = 0.f;
  bool have_r = false, have_w = false;
  for (uint32_t li = 0; li < h->n_local; ++li) {
    const LocalRank& L = h->lr[li];
    const ResultRow* row = L.row;
    const uint32_t g = L.grank;
    out->row_mask |= 1u << g;
    for (uint32_t j = 0; j < h->n_total; ++j) out->status[g * CDPROBE_MAX_GPUS + j] = h->status[g][j];
    if (!pl.diag) {
      out->reach_read[g * CDPROBE_MAX_GPUS + g] = 1;  // frozen oracle: reach[i][i] = 1 (SURVEY.md §8c)
      out->reach_write[g * CDPROBE_MAX_GPUS + g] = 1;
    }
    if (row->aborted) out->aborted = 1;
    out->device_ms[li] = row->t_last > row->t_first ? (double)(row->t_last - row->t_first) / 1e6 : 0.0;
    out->kernel_ms[li] = row->t_exit > row->t_enter ? (double)(row->t_exit - row->t_enter) / 1e6 : 0.0;
    double bar_ns = 0.0;
    bool slow[kMaxRanks] = {};
    for (uint32_t p = 0; p < L.n_phases; ++p) {
      const PhaseOut& o = row->ph[p];
      if (p + 1 < L.n_phases) {
        const PhaseOut& nx = row->ph[p + 1];
        if (nx.t_start > o.t_arrive) bar_ns += (double)(nx.t_start - o.t_arrive);
      }
      const Job& job = L.phases[p].job[0];
      if (job.kind != kJobRead && job.kind != kJobWrite) continue;
      const uint32_t idx = g * CDPROBE_MAX_GPUS + (uint32_t)job.peer;
      const bool done = o.code[0] == kCodeOk && o.t_end[0] > o.t_start;
      const float gbps = done ? (float)((double)pl.bpp / (double)(o.t_end[0] - o.t_start)) : 0.f;
      const bool offdiag = (uint32_t)job.peer != g || h->n_total == 1;
      if (job.kind == kJobRead) {
        const bool ok = done && o.sum[0] == o.exp_sum[0] && o.xr[0] == o.exp_xr[0];
        out->reach_read[idx] = ok ? 1 : 0;
        out->gbps_read[idx] = gbps;
        out->sum_read[idx] = o.sum[0];
        out->xor_read[idx] = o.xr[0];
        if (offdiag) {
          if (!have_r || gbps < min_r) min_r = gbps;
          have_r = true;
          if (ok && (uint32_t)job.peer != g && gbps < gate_r) slow[job.peer] = true;
        }
      } else {
        const bool ok = done && o.verdict[0] == h->launch_seq * 4ull + kVerdictOk;
        out->reach_write[idx] = ok ? 1 : 0;
        out->gbps_write[idx] = gbps;
        out->sum_write[idx] = o.sum[0];
        out->xor_write[idx] = o.xr[0];
        if (offdiag) {
          if (!have_w || gbps < min_w) min_w = gbps;
          have_w = true;
          if (ok && (uint32_t)job.peer != g && gbps < gate_w) slow[job.peer] = true;
        }
      }
    }
    out->barrier_us[li] = bar_ns / 1e3;
    // every off-diagonal cell of this row must have been probed, reachable and at speed
    for (uint32_t j = 0; j < h->n_total; ++j) {
      if (j == g) continue;
      // P2P is not applicable between MIG instances: the cell stays 0 but must not turn a MIG-only
      // domain NotReady (SURVEY H8)
      if (h->status[g][j] == CDPROBE_ERR_UNSUPPORTED || h->status[j][g] == CDPROBE_ERR_UNSUPPORTED) continue;
      const uint32_t idx = g * CDPROBE_MAX_GPUS + j;
      const bool unreachable = ((h->cfg.ops & CDPROBE_OP_READ) && !out->reach_read[idx]) ||
                               ((h->cfg.ops & CDPROBE_OP_WRITE) && !out->reach_write[idx]);
      if (unreachable) out->unreachable_pairs++;
      else if (slow[j]) out->slow_pairs++;
      if (unreachable || slow[j]) verdict = false;
    }
    if (h->n_total == 1 && pl.diag) {  // loop-back: reachability only (HBM speed is not a fabric property)
      const uint32_t idx = g * CDPROBE_MAX_GPUS + g;
      if (((h->cfg.ops & CDPROBE_OP_READ) && !out->reach_read[idx]) || ((h->cfg.ops & CDPROBE_OP_WRITE) && !out->reach_write[idx]))
        verdict = false;
    }
  }
  out->min_gbps_read = min_r;
  out->min_gbps_write = min_w;
  out->verdict = (verdict && !out->aborted) ? 1u : 0u;
}

// CDPROBE_OPT_LINK_COUNTERS, first enabling: one report row per distinct device of the local ranks, and NVML with a
// handle for each.
static int links_open(cdprobe* h) {
  h->links = new (std::nothrow) LinkCounters();
  if (h->links == nullptr) return CDPROBE_ERR_NOMEM;
  cdprobe_links_t& rep = h->links->report;
  char uuid[kMaxRanks][48] = {};
  bool mig[kMaxRanks] = {};
  uint32_t n = 0;
  for (uint32_t li = 0; li < h->n_local; ++li) {
    const LocalRank& L = h->lr[li];
    uint32_t d = 0;
    while (d < n && strncmp(uuid[d], L.uuid, 48) != 0) ++d;
    if (d == n) {
      memcpy(uuid[n], L.uuid, 48);
      mig[n++] = L.mig;
    }
    rep.dev[d].rank_mask |= 1u << L.grank;
  }
  for (uint32_t d = 0; d < n; ++d) memcpy(rep.dev[d].uuid, uuid[d], 48);
  h->links->sampler.open(n, uuid, mig);
  return CDPROBE_OK;
}

// The first sample of a run, before probe_ms's clock starts.
static void links_before(cdprobe* h) {
  LinkCounters& lc = *h->links;
  const double t = now_ms();
  lc.sampler.sample(lc.before, true);
  lc.before_ms = now_ms() - t;
}

// The second sample, after probe_ms's clock has stopped, and the report: the deltas next to the payload the run's
// phase tables moved between devices.
static void links_after(cdprobe* h, const cdprobe_result_t* out) {
  LinkCounters& lc = *h->links;
  const double t = now_ms();
  lc.sampler.sample(lc.after, false);
  cdprobe_links_t& rep = lc.report;
  rep.sample_ms = lc.before_ms + (now_ms() - t);
  rep.run_seq = h->launch_seq;
  rep.n_devices = lc.sampler.n();
  uint32_t dev[kMaxRanks];  // rank -> the lowest rank on the same device
  for (uint32_t r = 0; r < h->n_total; ++r) {
    dev[r] = r;
    for (uint32_t q = 0; q < r; ++q)
      if (strncmp(h->rank_uuid[q], h->rank_uuid[r], 48) == 0) {
        dev[r] = q;
        break;
      }
  }
  uint32_t ran = h->n_total >= 32 ? 0xffffffffu : (1u << h->n_total) - 1u;
  for (uint32_t li = 0; li < h->n_local; ++li)
    if (h->debug_skip_rank == li + 1 || (h->solo_rank != 0 && h->solo_rank != li + 1)) ran &= ~(1u << h->lr[li].grank);
  ScheduleInput in;
  in.plan = &h->plan;
  in.ops = h->cfg.ops;
  in.flags = h->cfg.flags;
  in.ctas = h->lr[0].ctas;
  in.verify_ctas = h->verify_ctas;
  in.status = h->status;
  uint64_t tx[kMaxRanks], rx[kMaxRanks];
  link_payload(in, ran, dev, out->warmed ? h->warm_bytes : 0, tx, rx);
  for (uint32_t d = 0; d < rep.n_devices; ++d) {
    cdprobe_link_device_t& row = rep.dev[d];
    link_delta(lc.before[d], lc.after[d], &row);
    const uint32_t r = dev[__builtin_ctz(row.rank_mask)];
    row.expected_tx_kib = tx[r] / 1024;
    row.expected_rx_kib = rx[r] / 1024;
  }
}

}  // namespace cdp

// ------------------------------------------------------------------ C ABI ----
extern "C" {

uint32_t cdprobe_abi_version(void) { return CDPROBE_ABI_VERSION; }

const char* cdprobe_strerror(int code) {
  switch (code) {
    case CDPROBE_OK: return "ok";
    case CDPROBE_ERR_ABI: return "ABI version mismatch";
    case CDPROBE_ERR_ARG: return "invalid argument";
    case CDPROBE_ERR_NO_DEVICE: return "no CUDA driver or device (there is no CPU fallback)";
    case CDPROBE_ERR_CUDA: return "CUDA call failed";
    case CDPROBE_ERR_TIMEOUT: return "probe timed out";
    case CDPROBE_ERR_RENDEZVOUS: return "multi-process rendezvous failed";
    case CDPROBE_ERR_NOMEM: return "out of memory";
    case CDPROBE_ERR_UNSUPPORTED: return "device or driver lacks a required feature";
    case CDPROBE_ERR_STATE: return "handle is in an unusable state";
    case CDPROBE_ERR_INTEGRITY: return "integrity self-check failed";
    default: return "unknown cdprobe error";
  }
}

const char* cdprobe_last_error(void) { return cdp::g_last_error.c_str(); }

int cdprobe_open(const cdprobe_config_t* cfg, cdprobe_t** out) {
  cdp::g_last_error.clear();
  if (cfg == nullptr || out == nullptr) return CDPROBE_ERR_ARG;
  *out = nullptr;
  if (cfg->abi != CDPROBE_ABI_VERSION) return CDPROBE_ERR_ABI;
  cdprobe* h = new (std::nothrow) cdprobe();
  if (h == nullptr) return CDPROBE_ERR_NOMEM;
  const int rc = cdp::open_impl(cfg, h);
  if (rc != CDPROBE_OK) {
    const std::string keep = cdp::g_last_error;
    cdp::destroy(h);
    cdp::g_last_error = keep;
    return rc;
  }
  *out = h;
  return CDPROBE_OK;
}

int cdprobe_run(cdprobe_t* h, cdprobe_result_t* out) {
  cdp::g_last_error.clear();
  if (h == nullptr || out == nullptr) return CDPROBE_ERR_ARG;
  // The caller reads *out whatever the return code (the daemon writes a verdict from it): never leave it
  // as it came in.
  memset(out, 0, sizeof(*out));
  out->abi = CDPROBE_ABI_VERSION;
  out->n = h->n_total;
  out->bytes_per_pair = h->plan.bpp;
  out->rounds = h->plan.rounds;
  if (const int rc = cdp::require_usable(h); rc != CDPROBE_OK) return rc;
  if (h->link_counters) cdp::links_before(h);  // before probe_ms: the samples are not part of the probe
  const double t0 = cdp::now_ms();
  h->launch_seq++;
  h->last_run_seq = h->launch_seq;
  out->run_seq = h->launch_seq;
  h->warm_now = h->warm_mode == 2 ||
                (h->warm_mode == 1 && (h->last_run_end_ms < 0 || t0 - h->last_run_end_ms > h->warm_idle_ms));
  cdp::ProbeParams P;
  for (uint32_t li = 0; li < h->n_local; ++li) {
    cdp::LocalRank& L = h->lr[li];
    const bool skipped = h->debug_skip_rank == li + 1 || (h->solo_rank != 0 && h->solo_rank != li + 1);
    if (skipped) {  // fault injection / solo profiling: this rank never shows up at the barriers
      memset(L.row->ph, 0, sizeof(L.row->ph));
      L.row->aborted = h->solo_rank ? 0u : 1u;
      L.row->n_phases = L.n_phases;
      L.row->t_first = L.row->t_last = 0;
      L.row->t_enter = L.row->t_exit = 0;
      L.row->done = h->launch_seq;
      continue;
    }
    if (h->solo_rank == li + 1) {
      // only this rank's own transfers; nobody to wait for, nobody verifies (reach_write stays 0)
      cdp::Phase solo[cdp::kMaxPhases];
      for (uint32_t p = 0; p < L.n_phases; ++p) {
        solo[p] = L.phases[p];
        solo[p].sync_mask = 0;
        solo[p].post_mask = 0;
        for (int jb = 0; jb < 2; ++jb)
          if (solo[p].job[jb].kind == cdp::kJobVerify) solo[p].job[jb].kind = cdp::kJobNone;
      }
      cdp::fill_params(h, li, solo, L.n_phases, 0u, &P);
    } else {
      cdp::fill_params(h, li, L.phases, L.n_phases, L.peer_mask, &P);
    }
    if (h->event_timing) {
      cudaSetDevice(L.ordinal);
      cudaEventRecord(L.ev0, L.stream);
    }
    const int rc = cdp::launch_one(h, li, P);
    if (rc != CDPROBE_OK) {
      h->sticky = true;
      return rc;
    }
    if (h->event_timing) cudaEventRecord(L.ev1, L.stream);
    out->launches++;
    out->phases = L.n_phases;
  }
  if (!cdp::wait_rows(h, h->launch_seq)) {
    h->sticky = true;
    if (cdp::g_last_error.empty()) cdp::set_err("host watchdog: kernels did not report within timeout_ms + 2 s");
    out->probe_ms = cdp::now_ms() - t0;
    return CDPROBE_ERR_TIMEOUT;
  }
  cdp::assemble(h, out);
  h->last_run_end_ms = cdp::now_ms();
  out->probe_ms = h->last_run_end_ms - t0;
  h->last_probe_ms = out->probe_ms;
  out->warmed = (h->warm_now && h->plan.rounds > 0) ? 1u : 0u;  // N = 1 has no link to wake
  if (h->event_timing) {  // after probe_ms: the event round trip is not part of the probe
    for (uint32_t li = 0; li < h->n_local; ++li) {
      cdp::LocalRank& L = h->lr[li];
      if (h->debug_skip_rank == li + 1 || (h->solo_rank != 0 && h->solo_rank != li + 1)) continue;
      float ms = 0.f;
      cudaSetDevice(L.ordinal);
      if (cudaEventSynchronize(L.ev1) == cudaSuccess && cudaEventElapsedTime(&ms, L.ev0, L.ev1) == cudaSuccess)
        out->event_ms[li] = ms;
    }
  }
  if (h->link_counters) cdp::links_after(h, out);
  if (out->aborted) {
    for (uint32_t li = 0; li < h->n_local; ++li) {
      const int rc = cdp::reset_ctrl_local(h, li);
      if (rc != CDPROBE_OK) {
        h->sticky = true;
        return rc;
      }
    }
    cdp::set_err("device watchdog fired (a peer did not reach a barrier within timeout_ms)");
    // In one process all ranks share the run counter and the handle stays usable.  Across processes
    // the peers' counters may have diverged: the handle must be reopened.
    if (h->cfg.world_size > 1) h->sticky = true;
    return CDPROBE_ERR_TIMEOUT;
  }
  return CDPROBE_OK;
}

int cdprobe_gather(cdprobe_t* h, cdprobe_result_t* inout) {
  if (h == nullptr || inout == nullptr) return CDPROBE_ERR_ARG;
  if (h->cfg.world_size <= 1) return CDPROBE_OK;
  std::vector<cdprobe_result_t> all(h->cfg.world_size);
  std::string err;
  if (h->rdv.allgather(inout, sizeof(cdprobe_result_t), all.data(), &err) != 0) {
    cdp::set_err(err);
    return CDPROBE_ERR_RENDEZVOUS;
  }
  for (uint32_t r = 0; r < h->cfg.world_size; ++r) {
    if (r == h->cfg.rank) continue;
    const cdprobe_result_t& o = all[r];
    for (uint32_t g = 0; g < h->n_total; ++g) {
      if (!((o.row_mask >> g) & 1u) || ((inout->row_mask >> g) & 1u)) continue;
      const size_t a = (size_t)g * CDPROBE_MAX_GPUS;
      memcpy(inout->reach_read + a, o.reach_read + a, CDPROBE_MAX_GPUS);
      memcpy(inout->reach_write + a, o.reach_write + a, CDPROBE_MAX_GPUS);
      memcpy(inout->gbps_read + a, o.gbps_read + a, CDPROBE_MAX_GPUS * sizeof(float));
      memcpy(inout->gbps_write + a, o.gbps_write + a, CDPROBE_MAX_GPUS * sizeof(float));
      memcpy(inout->status + a, o.status + a, CDPROBE_MAX_GPUS * sizeof(int32_t));
      memcpy(inout->sum_read + a, o.sum_read + a, CDPROBE_MAX_GPUS * sizeof(uint64_t));
      memcpy(inout->xor_read + a, o.xor_read + a, CDPROBE_MAX_GPUS * sizeof(uint64_t));
      memcpy(inout->sum_write + a, o.sum_write + a, CDPROBE_MAX_GPUS * sizeof(uint64_t));
      memcpy(inout->xor_write + a, o.xor_write + a, CDPROBE_MAX_GPUS * sizeof(uint64_t));
      inout->row_mask |= 1u << g;
    }
    if (!o.verdict) inout->verdict = 0;
    if (o.aborted) inout->aborted = 1;
    inout->unreachable_pairs += o.unreachable_pairs;
    inout->slow_pairs += o.slow_pairs;
    if (o.min_gbps_read > 0.f && (inout->min_gbps_read == 0.f || o.min_gbps_read < inout->min_gbps_read))
      inout->min_gbps_read = o.min_gbps_read;
    if (o.min_gbps_write > 0.f && (inout->min_gbps_write == 0.f || o.min_gbps_write < inout->min_gbps_write))
      inout->min_gbps_write = o.min_gbps_write;
    if (o.probe_ms > inout->probe_ms) inout->probe_ms = o.probe_ms;
  }
  return CDPROBE_OK;
}

int cdprobe_info(cdprobe_t* h, cdprobe_info_t* out) {
  if (h == nullptr || out == nullptr) return CDPROBE_ERR_ARG;
  memset(out, 0, sizeof(*out));
  out->abi = CDPROBE_ABI_VERSION;
  out->n = h->n_total;
  out->n_local = h->n_local;
  out->first_local_rank = h->first;
  for (uint32_t li = 0; li < h->n_local; ++li) {
    const cdp::LocalRank& L = h->lr[li];
    out->ordinal[li] = L.ordinal;
    out->sm_count[li] = (uint32_t)L.sm_count;
    out->ctas[li] = L.ctas;
    out->mig[li] = L.mig ? 1u : 0u;
    memcpy(out->uuid[li], L.uuid, sizeof(out->uuid[li]));
    for (uint32_t s = 0; s < h->plan.n_slices; ++s) {
      out->src_sum[li][s] = h->src_sum[li][s];
      out->src_xor[li][s] = h->src_xor[li][s];
    }
  }
  out->handle_type = h->handle_type;
  out->path = h->path;
  out->bytes_per_pair = h->plan.bpp;
  out->alloc_bytes = h->plan.alloc_bytes;
  out->n_slices = h->plan.n_slices;
  out->smem_bytes = cdp::kSmemBytes;
  out->open_ms = h->open_ms;
  out->fill_ms = h->fill_ms;
  return CDPROBE_OK;
}

int cdprobe_trace(cdprobe_t* h, uint32_t local, cdprobe_trace_t* out) {
  if (h == nullptr || out == nullptr || local >= h->n_local) return CDPROBE_ERR_ARG;
  memset(out, 0, sizeof(*out));
  out->abi = CDPROBE_ABI_VERSION;
  const cdp::LocalRank& L = h->lr[local];
  const cdp::ResultRow* row = L.row;
  out->n_phases = L.n_phases;
  const uint64_t t0 = row->t_first;
  auto rel = [&](uint64_t t) { return t > t0 ? t - t0 : 0ull; };
  for (uint32_t p = 0; p < L.n_phases; ++p) {
    const cdp::PhaseOut& o = row->ph[p];
    out->kind0[p] = L.phases[p].job[0].kind;
    out->kind1[p] = L.phases[p].job[1].kind;
    out->peer0[p] = L.phases[p].job[0].peer;
    out->peer1[p] = L.phases[p].job[1].peer;
    out->sync_mask[p] = (uint16_t)(L.phases[p].sync_mask & L.peer_mask);
    out->post_mask[p] = (uint16_t)(L.phases[p].post_mask & L.peer_mask);
    out->sync_all[p] = (uint8_t)(L.peer_mask != 0 && (L.phases[p].sync_mask & L.peer_mask) == L.peer_mask);
    out->t_start[p] = rel(o.t_start);
    out->t_end0[p] = rel(o.t_end[0]);
    out->t_end1[p] = rel(o.t_end[1]);
    out->t_arrive[p] = rel(o.t_arrive);
  }
  return CDPROBE_OK;
}

int cdprobe_set_option(cdprobe_t* h, uint32_t option, uint64_t value) {
  if (h == nullptr) return CDPROBE_ERR_ARG;
  for (const cdp::FaultOption& o : cdp::kFaultOptions) {
    if (o.option == option) {
      h->meas[o.meas].fault = value;
      return CDPROBE_OK;
    }
  }
  switch (option) {
    case CDPROBE_OPT_EVENT_TIMING:
      h->event_timing = value != 0;
      return CDPROBE_OK;
    case CDPROBE_OPT_CTAS:
      // a value truncated to 32 bits could become 0 CTAs: a grid no launch accepts
      if (value > UINT32_MAX) return CDPROBE_ERR_ARG;
      for (uint32_t li = 0; li < h->n_local; ++li) {
        cdp::LocalRank& L = h->lr[li];
        uint32_t c = value ? (uint32_t)value : (uint32_t)L.sm_count;
        if (c > (uint32_t)L.max_ctas) c = (uint32_t)L.max_ctas;
        L.ctas = c;
      }
      return cdp::rebuild_all(h);
    case CDPROBE_OPT_PATH:
      if (value > 2) return CDPROBE_ERR_ARG;
      h->path = (uint32_t)value;
      return CDPROBE_OK;
    case CDPROBE_OPT_TIMEOUT_MS:
      if (value == 0 || value > 600000) return CDPROBE_ERR_ARG;
      h->cfg.timeout_ms = (uint32_t)value;
      return CDPROBE_OK;
    case CDPROBE_OPT_OVERLAP_VERIFY:
      return cdp::set_flag(h, CDPROBE_FLAG_OVERLAP_VERIFY, value != 0);
    case CDPROBE_OPT_UNIDIRECTIONAL:
      return cdp::set_flag(h, CDPROBE_FLAG_UNIDIRECTIONAL, value != 0);
    case CDPROBE_OPT_ALL_RANK_BARRIERS:
      return cdp::set_flag(h, CDPROBE_FLAG_ALL_RANK_BARRIERS, value != 0);
    case CDPROBE_OPT_PAIR_BARRIERS:
      return cdp::set_flag(h, CDPROBE_FLAG_PAIR_BARRIERS, value != 0);
    case CDPROBE_OPT_CTAS_RANK:
    {
      const uint64_t li = value >> 16;  // not truncated: stray high bits must not name another rank
      const uint32_t c = (uint32_t)(value & 0xffffu);
      if (li == 0 || li > h->n_local || c == 0) return CDPROBE_ERR_ARG;
      cdp::LocalRank& L = h->lr[li - 1];
      L.ctas = c > (uint32_t)L.max_ctas ? (uint32_t)L.max_ctas : c;
      return cdp::rebuild_all(h);
    }
    case CDPROBE_OPT_MIN_FRACTION_PPM:
      if (value > 100000000ull) return CDPROBE_ERR_ARG;
      h->cfg.min_fraction = (float)((double)value / 1e6);
      return CDPROBE_OK;
    case CDPROBE_OPT_LINK_PEAK_MBPS:
      if (value > 100000000000ull) return CDPROBE_ERR_ARG;
      h->cfg.link_peak_gbps = (float)((double)value / 1e3);
      return CDPROBE_OK;
    case CDPROBE_OPT_SOLO_RANK:
      if (value > h->n_local || h->cfg.world_size > 1) return CDPROBE_ERR_ARG;
      h->solo_rank = (uint32_t)value;
      return CDPROBE_OK;
    case CDPROBE_OPT_DEBUG_SKIP_RANK:
      if (value > h->n_local) return CDPROBE_ERR_ARG;
      h->debug_skip_rank = (uint32_t)value;
      return CDPROBE_OK;
    case CDPROBE_OPT_WARMUP:
      if (value > 2) return CDPROBE_ERR_ARG;
      h->warm_mode = (uint32_t)value;
      return CDPROBE_OK;
    case CDPROBE_OPT_WARMUP_BYTES:
      h->warm_bytes = value / 128 * 128;
      return CDPROBE_OK;
    case CDPROBE_OPT_VERIFY_CTAS:
      if (value == 0 || value > 65535) return CDPROBE_ERR_ARG;
      h->verify_ctas = (uint32_t)value;
      return cdp::rebuild_all(h);
    case CDPROBE_OPT_LINK_COUNTERS:
      if (value > 1) return CDPROBE_ERR_ARG;
      if (value != 0 && h->links == nullptr)
        if (const int rc = cdp::links_open(h); rc != CDPROBE_OK) return rc;
      h->link_counters = value != 0;
      return CDPROBE_OK;
    default:
      return CDPROBE_ERR_ARG;
  }
}

int cdprobe_unmap_peer(cdprobe_t* h, uint32_t local, uint32_t peer) {
  if (h == nullptr || local >= h->n_local || peer >= h->n_total) return CDPROBE_ERR_ARG;
  if (h->cfg.world_size > 1) return CDPROBE_ERR_UNSUPPORTED;  // peers would not learn about it
  const uint32_t g = h->lr[local].grank;
  if (peer == g) return CDPROBE_ERR_ARG;
  cdp::unmap_peer(h, h->mem, local, peer);
  h->status[g][peer] = cdp::kStatusUnmapped;
  return cdp::rebuild_all(h);
}

int cdprobe_remap_peer(cdprobe_t* h, uint32_t local, uint32_t peer) {
  if (h == nullptr || local >= h->n_local || peer >= h->n_total) return CDPROBE_ERR_ARG;
  const uint32_t g = h->lr[local].grank;
  if (peer == g) return CDPROBE_ERR_ARG;
  if (const int rc = cdp::require_usable(h); rc != CDPROBE_OK) return rc;
  cdp::unmap_peer(h, h->mem, local, peer);
  const int32_t st = cdp::map_peer(h, h->mem, local, peer);
  if (st != 0 && h->cfg.world_size > 1) {
    // the other processes build their phase tables from the mapping status exchanged at open and would
    // not learn that this pair is gone: the domain has to be reopened
    h->sticky = true;
    cdp::set_err("re-mapping a peer failed in a multi-process domain: " + h->drv.error_name((CUresult)st));
    return CDPROBE_ERR_CUDA;
  }
  h->status[g][peer] = st;
  const int rc = cdp::rebuild_all(h);
  if (rc != CDPROBE_OK) return rc;
  return st == 0 ? CDPROBE_OK : CDPROBE_ERR_CUDA;
}

int cdprobe_corrupt(cdprobe_t* h, uint32_t local, uint64_t byte_offset, uint64_t xor_mask) {
  if (h == nullptr || local >= h->n_local) return CDPROBE_ERR_ARG;
  if (byte_offset % 8 != 0 || byte_offset + 8 > h->plan.src_bytes) return CDPROBE_ERR_ARG;
  cdp::LocalRank& L = h->lr[local];
  CDP_RT(cudaSetDevice(L.ordinal));
  uint8_t* p = reinterpret_cast<uint8_t*>(h->mem.va[local][L.grank]) + h->plan.src_off + byte_offset;
  uint64_t w = 0;
  CDP_RT(cudaMemcpyAsync(&w, p, 8, cudaMemcpyDeviceToHost, L.stream));
  CDP_RT(cudaStreamSynchronize(L.stream));
  w ^= xor_mask;
  CDP_RT(cudaMemcpyAsync(p, &w, 8, cudaMemcpyHostToDevice, L.stream));
  CDP_RT(cudaStreamSynchronize(L.stream));
  return CDPROBE_OK;
}

int cdprobe_corrupt_landing(cdprobe_t* h, uint32_t local, uint32_t target, uint32_t n, const uint64_t* word,
                            const uint64_t* xor_mask) {
  cdp::g_last_error.clear();
  if (h == nullptr || local >= h->n_local || target >= h->n_total || n > cdp::kMaxLandingFaults) return CDPROBE_ERR_ARG;
  if (n > 0 && (word == nullptr || xor_mask == nullptr)) return CDPROBE_ERR_ARG;
  const uint32_t g = h->lr[local].grank;
  const uint64_t words = h->plan.bpp / 8;
  cdp::LandingFault f;
  memset(&f, 0, sizeof(f));
  f.n = n;
  f.target = target;
  for (uint32_t e = 0; e < n; ++e) {
    if (word[e] >= words || xor_mask[e] == 0) return CDPROBE_ERR_ARG;
    for (uint32_t q = 0; q < e; ++q)
      if (word[q] == word[e]) return CDPROBE_ERR_ARG;
    f.word[e] = word[e];
    f.mask[e] = xor_mask[e];
  }
  if (n > 0 && target == g && !h->plan.diag) {
    cdp::set_err("cell (i, i) exists only with a loop-back slot (n == 1 or CDPROBE_FLAG_LOCAL_DIAG)");
    return CDPROBE_ERR_ARG;
  }
  if (const int rc = cdp::require_usable(h); rc != CDPROBE_OK) return rc;
  if (n > 0 && cdp::cell_status(h, local, target) != 0) {
    cdp::set_err("the issuer does not map the target");
    return CDPROBE_ERR_STATE;
  }
  // one armed cell per handle: clear the previous one, wherever it is
  if (h->fault_local >= 0) {
    cdp::LandingFault off;
    memset(&off, 0, sizeof(off));
    const int rc = cdp::write_fault(h, (uint32_t)h->fault_local, off);
    if (rc != CDPROBE_OK) return rc;
    h->fault_local = -1;
  }
  if (n == 0) return CDPROBE_OK;
  const int rc = cdp::write_fault(h, local, f);
  if (rc != CDPROBE_OK) return rc;
  h->fault_local = (int32_t)local;
  return CDPROBE_OK;
}

int cdprobe_ce_copy(cdprobe_t* h, uint32_t n_copies, const uint32_t* local, const uint32_t* peer, uint32_t push,
                    uint64_t bytes, uint32_t reps, double* ms_out) {
  cdp::g_last_error.clear();
  if (h == nullptr || local == nullptr || peer == nullptr || ms_out == nullptr || n_copies == 0 ||
      n_copies > h->n_local || reps == 0 || reps > 1024)
    return CDPROBE_ERR_ARG;
  if (const int rc = cdp::require_usable(h); rc != CDPROBE_OK) return rc;
  const cdp::Plan& pl = h->plan;
  uint64_t nb = bytes;
  if (nb == 0 || nb > pl.src_bytes) nb = pl.src_bytes;
  if (nb > pl.land_bytes) nb = pl.land_bytes;
  for (uint32_t k = 0; k < n_copies; ++k) {
    if (local[k] >= h->n_local || peer[k] >= h->n_total) return CDPROBE_ERR_ARG;
    for (uint32_t q = 0; q < k; ++q)
      if (local[q] == local[k]) return CDPROBE_ERR_ARG;  // one copy per local rank: each has one stream and event pair
    if (!h->mem.mapped[local[k]][peer[k]]) {
      cdp::set_err("peer is not mapped into this rank's address space");
      return CDPROBE_ERR_STATE;
    }
  }
  for (uint32_t k = 0; k < n_copies; ++k) {
    cdp::LocalRank& L = h->lr[local[k]];
    CDP_RT(cudaSetDevice(L.ordinal));
    const uint8_t* mine = reinterpret_cast<const uint8_t*>(h->mem.va[local[k]][L.grank]);
    const uint8_t* theirs = reinterpret_cast<const uint8_t*>(h->mem.va[local[k]][peer[k]]);
    const void* src = push ? mine + pl.src_off : theirs + pl.src_off;
    void* dst = const_cast<uint8_t*>(push ? theirs : mine) + pl.land_off;
    CDP_RT(cudaEventRecord(L.ev0, L.stream));
    for (uint32_t r = 0; r < reps; ++r) CDP_RT(cudaMemcpyAsync(dst, src, nb, cudaMemcpyDeviceToDevice, L.stream));
    CDP_RT(cudaEventRecord(L.ev1, L.stream));
  }
  for (uint32_t k = 0; k < n_copies; ++k) {
    cdp::LocalRank& L = h->lr[local[k]];
    CDP_RT(cudaSetDevice(L.ordinal));
    CDP_RT(cudaEventSynchronize(L.ev1));
    float ms = 0.f;
    CDP_RT(cudaEventElapsedTime(&ms, L.ev0, L.ev1));
    ms_out[k] = ms;
  }
  return CDPROBE_OK;
}

int cdprobe_gate(const cdprobe_config_t* cfg, uint32_t n_total, float* gate_read_gbps, float* gate_write_gbps) {
  if (cfg == nullptr || gate_read_gbps == nullptr || gate_write_gbps == nullptr) return CDPROBE_ERR_ARG;
  if (cfg->abi != CDPROBE_ABI_VERSION) return CDPROBE_ERR_ABI;
  if (cfg->link_peak_gbps < 0.f || cfg->min_fraction < 0.f) return CDPROBE_ERR_ARG;
  cdp::Plan pl;
  const int rc = cdp::make_plan(n_total, cfg->bytes, cfg->mode, cfg->flags, &pl);
  if (rc != CDPROBE_OK) return rc;
  *gate_read_gbps = cdp::gate_gbps_for(*cfg, n_total, pl.bpp, true);
  *gate_write_gbps = cdp::gate_gbps_for(*cfg, n_total, pl.bpp, false);
  return CDPROBE_OK;
}

int cdprobe_links(cdprobe_t* h, cdprobe_links_t* out) {
  if (h == nullptr || out == nullptr) return CDPROBE_ERR_ARG;
  if (h->links != nullptr && h->links->report.run_seq != 0) *out = h->links->report;
  else memset(out, 0, sizeof(*out));
  out->abi = CDPROBE_ABI_VERSION;
  return CDPROBE_OK;
}

void cdprobe_close(cdprobe_t* h) { cdp::destroy(h); }

}  // extern "C"
