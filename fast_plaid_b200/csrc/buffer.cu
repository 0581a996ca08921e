// Growable device buffers (fpb_buffer_*): a range of virtual addresses reserved once, backed by physical memory
// mapped in granules as it is committed, so that an index's arrays grow in place and their address never changes.
#include <mutex>
#include <vector>

#include <cuda.h>

#include "kernels.h"

namespace {

// The driver's virtual memory management, resolved at run time like cuTensorMapEncodeTiled (no link against
// libcuda).
struct Vmm {
  decltype(&cuMemAddressReserve) reserve = nullptr;
  decltype(&cuMemAddressFree) address_free = nullptr;
  decltype(&cuMemCreate) create = nullptr;
  decltype(&cuMemRelease) release = nullptr;
  decltype(&cuMemMap) map = nullptr;
  decltype(&cuMemUnmap) unmap = nullptr;
  decltype(&cuMemSetAccess) set_access = nullptr;
  decltype(&cuMemGetAllocationGranularity) granularity = nullptr;
  bool ok = false;
};

template <class T>
bool resolve(const char* name, T& fn) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || !p ||
      q != cudaDriverEntryPointSuccess) {
    cudaGetLastError();
    return false;
  }
  fn = reinterpret_cast<T>(p);
  return true;
}

const Vmm& vmm() {
  static Vmm v;
  static std::once_flag once;
  std::call_once(once, [] {
    v.ok = resolve("cuMemAddressReserve", v.reserve) && resolve("cuMemAddressFree", v.address_free) &&
           resolve("cuMemCreate", v.create) && resolve("cuMemRelease", v.release) && resolve("cuMemMap", v.map) &&
           resolve("cuMemUnmap", v.unmap) && resolve("cuMemSetAccess", v.set_access) &&
           resolve("cuMemGetAllocationGranularity", v.granularity);
  });
  return v;
}

int vmm_error(const char* what, CUresult r) {
  fpb_set_error("%s failed (CUresult %d)", what, int(r));
  return FPB_ERR_CUDA;
}

CUmemAllocationProp device_prop(int device) {
  CUmemAllocationProp p = {};
  p.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  p.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  p.location.id = device;
  return p;
}

}  // namespace

struct fpb_buffer {
  int device;
  CUdeviceptr base;
  size_t reserved;  // bytes of address space
  size_t granule;   // physical memory is mapped in multiples of this
  size_t mapped;    // bytes mapped from base
  std::vector<std::pair<CUmemGenericAllocationHandle, size_t>> chunks;  // in address order
  std::mutex mu;
};

constexpr size_t FPB_BUFFER_GRANULE = size_t(2) << 20;

extern "C" int fpb_buffer_reserve(fpb_buffer** out, int device, size_t max_bytes) {
  if (!out) {
    fpb_set_error("fpb_buffer_reserve: out is NULL");
    return FPB_ERR_INVALID;
  }
  *out = nullptr;
  if (device < 0) {
    fpb_set_error("fpb_buffer_reserve: device %d", device);
    return FPB_ERR_INVALID;
  }
  FPB_CUDA_CHECK(cudaSetDevice(device));
  FPB_CUDA_CHECK(cudaFree(nullptr));  // the primary context, current on this thread
  const Vmm& v = vmm();
  if (!v.ok) {
    fpb_set_error("fpb_buffer_reserve: the driver's virtual memory management entry points are unavailable");
    return FPB_ERR_UNSUPPORTED;
  }
  const CUmemAllocationProp prop = device_prop(device);
  size_t g = 0;
  CUresult r = v.granularity(&g, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM);
  if (r != CUDA_SUCCESS) return vmm_error("cuMemGetAllocationGranularity", r);
  const size_t granule = (FPB_BUFFER_GRANULE + g - 1) / g * g;
  if (max_bytes == 0) {  // up to the device's memory: a buffer can never need more
    size_t free_b = 0, total_b = 0;
    FPB_CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
    max_bytes = total_b;
  }
  const size_t reserved = (max_bytes + granule - 1) / granule * granule;
  CUdeviceptr base = 0;
  r = v.reserve(&base, reserved, granule, 0, 0);
  if (r != CUDA_SUCCESS) return vmm_error("cuMemAddressReserve", r);
  fpb_buffer* b = new fpb_buffer();
  b->device = device;
  b->base = base;
  b->reserved = reserved;
  b->granule = granule;
  b->mapped = 0;
  *out = b;
  return FPB_OK;
}

extern "C" int fpb_buffer_commit(fpb_buffer* b, size_t bytes) {
  if (!b) {
    fpb_set_error("fpb_buffer_commit: NULL buffer");
    return FPB_ERR_INVALID;
  }
  std::lock_guard<std::mutex> lock(b->mu);
  if (bytes <= b->mapped) return FPB_OK;
  if (bytes > b->reserved) {
    fpb_set_error("fpb_buffer_commit: %zu bytes exceed the %zu reserved", bytes, b->reserved);
    return FPB_ERR_INVALID;
  }
  FPB_CUDA_CHECK(cudaSetDevice(b->device));
  const Vmm& v = vmm();
  const size_t grow = (bytes - b->mapped + b->granule - 1) / b->granule * b->granule;
  const CUmemAllocationProp prop = device_prop(b->device);
  CUmemGenericAllocationHandle h;
  CUresult r = v.create(&h, grow, &prop, 0);
  if (r != CUDA_SUCCESS) {
    fpb_set_error("fpb_buffer_commit: cuMemCreate of %zu bytes failed (CUresult %d)", grow, int(r));
    return FPB_ERR_CUDA;
  }
  const CUdeviceptr at = b->base + b->mapped;
  r = v.map(at, grow, 0, h, 0);
  if (r != CUDA_SUCCESS) {
    v.release(h);
    return vmm_error("cuMemMap", r);
  }
  CUmemAccessDesc acc = {};
  acc.location = prop.location;
  acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  r = v.set_access(at, grow, &acc, 1);
  if (r != CUDA_SUCCESS) {
    v.unmap(at, grow);
    v.release(h);
    return vmm_error("cuMemSetAccess", r);
  }
  b->chunks.emplace_back(h, grow);
  b->mapped += grow;
  return FPB_OK;
}

extern "C" void* fpb_buffer_ptr(const fpb_buffer* b) { return b ? reinterpret_cast<void*>(b->base) : nullptr; }

extern "C" size_t fpb_buffer_mapped_bytes(const fpb_buffer* b) { return b ? b->mapped : 0; }

extern "C" void fpb_buffer_destroy(fpb_buffer* b) {
  if (!b) return;
  const Vmm& v = vmm();
  int prev = -1;
  const bool have_prev = cudaGetDevice(&prev) == cudaSuccess;
  cudaSetDevice(b->device);
  CUdeviceptr at = b->base;
  for (const auto& c : b->chunks) {
    v.unmap(at, c.second);
    v.release(c.first);
    at += c.second;
  }
  v.address_free(b->base, b->reserved);
  if (have_prev) cudaSetDevice(prev);
  delete b;
}
