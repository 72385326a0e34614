// vmm.cc — see vmm.h.
#include "vmm.h"

namespace cdp {

namespace {
template <typename Fn>
cudaError_t resolve(const char* name, Fn* out, std::string* err) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
  cudaError_t e = cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q);
  if (e != cudaSuccess) {
    if (err) *err = std::string("cudaGetDriverEntryPoint(") + name + "): " + cudaGetErrorString(e);
    return e;
  }
  if (q != cudaDriverEntryPointSuccess || p == nullptr) {
    if (err) *err = std::string("driver entry point not available: ") + name;
    return cudaErrorNotSupported;
  }
  *out = reinterpret_cast<Fn>(p);
  return cudaSuccess;
}
}  // namespace

cudaError_t Driver::load(std::string* err) {
  cudaError_t e;
#define CDP_RESOLVE(field, sym)                                       \
  if ((e = resolve(sym, &field, err)) != cudaSuccess) return e;
  CDP_RESOLVE(MemCreate, "cuMemCreate")
  CDP_RESOLVE(MemRelease, "cuMemRelease")
  CDP_RESOLVE(MemAddressReserve, "cuMemAddressReserve")
  CDP_RESOLVE(MemAddressFree, "cuMemAddressFree")
  CDP_RESOLVE(MemMap, "cuMemMap")
  CDP_RESOLVE(MemUnmap, "cuMemUnmap")
  CDP_RESOLVE(MemSetAccess, "cuMemSetAccess")
  CDP_RESOLVE(MemGetAllocationGranularity, "cuMemGetAllocationGranularity")
  CDP_RESOLVE(MemExportToShareableHandle, "cuMemExportToShareableHandle")
  CDP_RESOLVE(MemImportFromShareableHandle, "cuMemImportFromShareableHandle")
  CDP_RESOLVE(GetErrorName, "cuGetErrorName")
#undef CDP_RESOLVE
  return cudaSuccess;
}

bool Driver::load_multicast() {
  if (multicast < 0)
    multicast = resolve("cuMulticastCreate", &MulticastCreate, nullptr) == cudaSuccess &&
                resolve("cuMulticastAddDevice", &MulticastAddDevice, nullptr) == cudaSuccess &&
                resolve("cuMulticastBindMem", &MulticastBindMem, nullptr) == cudaSuccess &&
                resolve("cuMulticastUnbind", &MulticastUnbind, nullptr) == cudaSuccess &&
                resolve("cuMulticastGetGranularity", &MulticastGetGranularity, nullptr) == cudaSuccess &&
                resolve("cuDeviceGet", &DeviceGet, nullptr) == cudaSuccess &&
                resolve("cuDeviceGetAttribute", &DeviceGetAttribute, nullptr) == cudaSuccess;
  return multicast == 1;
}

cudaError_t Driver::load_stream_wait(std::string* err) {
  return StreamWaitValue64 != nullptr ? cudaSuccess : resolve("cuStreamWaitValue64", &StreamWaitValue64, err);
}

cudaError_t Driver::load_stream_write(std::string* err) {
  return StreamWriteValue64 != nullptr ? cudaSuccess : resolve("cuStreamWriteValue64", &StreamWriteValue64, err);
}

std::string Driver::error_name(CUresult r) const {
  const char* s = nullptr;
  if (GetErrorName && GetErrorName(r, &s) == CUDA_SUCCESS && s) return s;
  return "CUresult(" + std::to_string((int)r) + ")";
}

}  // namespace cdp
