// vmm.h — CUDA driver entry points used for the probe allocations.
//
// libcdprobe.so links only the static CUDA runtime; libcuda.so.1 is reached
// lazily through cudaGetDriverEntryPoint, the same late-binding idea go-nvml
// uses for libnvidia-ml.so.1 (vendor/github.com/NVIDIA/go-nvml/pkg/nvml/lib.go:29-80),
// so the daemon binary starts on nodes without a driver and fails loudly
// (CDPROBE_ERR_NO_DEVICE) only when a probe is opened.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <string>

namespace cdp {

struct Driver {
  CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
  CUresult (*MemRelease)(CUmemGenericAllocationHandle) = nullptr;
  CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
  CUresult (*MemAddressFree)(CUdeviceptr, size_t) = nullptr;
  CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
  CUresult (*MemUnmap)(CUdeviceptr, size_t) = nullptr;
  CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
  CUresult (*MemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
  CUresult (*MemExportToShareableHandle)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType,
                                         unsigned long long) = nullptr;
  CUresult (*MemImportFromShareableHandle)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType) = nullptr;
  CUresult (*GetErrorName)(CUresult, const char**) = nullptr;
  // Multicast objects (cdprobe_allreduce_nvls): resolved by load_multicast, apart from load's set, so that a driver
  // without them still opens a handle.
  CUresult (*MulticastCreate)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*) = nullptr;
  CUresult (*MulticastAddDevice)(CUmemGenericAllocationHandle, CUdevice) = nullptr;
  CUresult (*MulticastBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t,
                               unsigned long long) = nullptr;
  CUresult (*MulticastUnbind)(CUmemGenericAllocationHandle, CUdevice, size_t, size_t) = nullptr;
  CUresult (*MulticastGetGranularity)(size_t*, const CUmulticastObjectProp*, CUmulticastGranularity_flags) = nullptr;
  CUresult (*DeviceGet)(CUdevice*, int) = nullptr;
  CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice) = nullptr;
  int multicast = -1;  // load_multicast's verdict, -1: not asked yet
  // The stream wait of cdprobe_memcpy: resolved by load_stream_wait on its first call, apart from load's set.
  CUresult (*StreamWaitValue64)(CUstream, CUdeviceptr, cuuint64_t, unsigned int) = nullptr;
  // The stream write of cdprobe_ce_alltoall: resolved by load_stream_write on its first call, apart from load's set.
  CUresult (*StreamWriteValue64)(CUstream, CUdeviceptr, cuuint64_t, unsigned int) = nullptr;

  // Returns cudaSuccess or the runtime error that prevented loading.
  cudaError_t load(std::string* err);
  // Whether every multicast entry point above resolved; asked once.
  bool load_multicast();
  // Resolves StreamWaitValue64 once; returns cudaSuccess or why it is missing.
  cudaError_t load_stream_wait(std::string* err);
  // Resolves StreamWriteValue64 once; returns cudaSuccess or why it is missing.
  cudaError_t load_stream_write(std::string* err);
  std::string error_name(CUresult r) const;
};

}  // namespace cdp
