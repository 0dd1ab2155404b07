// cuda_emu_pointer.h -- cudaPointerGetAttributes for the CPU emulation of the CUDA runtime (cuda_emu.h), TEST
// INFRASTRUCTURE ONLY.  The emulation build of the library (build_emu_lib.py) includes it into b200z_api.cu, whose
// *_to_device decode batches ask whether the caller's output base is device memory.
//
// "Device" memory is host memory in the emulation, so every address counts as device memory except the page-locked
// blocks of this translation unit's cudaHostAlloc (b200z_host_alloc among them): those are host memory, which is what a
// test passes as a host pointer.
#pragma once
#include <iterator>
#include <map>
#include <mutex>

#include "cuda_emu.h"

enum cudaMemoryType { cudaMemoryTypeUnregistered = 0, cudaMemoryTypeHost = 1, cudaMemoryTypeDevice = 2, cudaMemoryTypeManaged = 3 };
struct cudaPointerAttributes {
  cudaMemoryType type;
  int device;
  void *devicePointer, *hostPointer;
};

namespace cuemu {
inline std::map<uintptr_t, size_t> &host_blocks() {
  static std::map<uintptr_t, size_t> m;
  return m;
}
inline std::mutex &host_blocks_mutex() {
  static std::mutex m;
  return m;
}
template <typename T>
static inline cudaError_t host_alloc_tracked(T **p, size_t n, unsigned flags) {
  const cudaError_t e = cudaHostAlloc((void **)p, n, flags);
  if (e == cudaSuccess) {
    std::lock_guard<std::mutex> lk(host_blocks_mutex());
    host_blocks()[(uintptr_t)*p] = n ? n : 1;
  }
  return e;
}
static inline cudaError_t free_host_tracked(void *p) {
  {
    std::lock_guard<std::mutex> lk(host_blocks_mutex());
    host_blocks().erase((uintptr_t)p);
  }
  return cudaFreeHost(p);
}
}  // namespace cuemu

static inline cudaError_t cudaPointerGetAttributes(cudaPointerAttributes *a, const void *p) {
  std::lock_guard<std::mutex> lk(cuemu::host_blocks_mutex());
  const auto &m = cuemu::host_blocks();
  const auto it = m.upper_bound((uintptr_t)p);
  const bool host = it != m.begin() && (uintptr_t)p < std::prev(it)->first + std::prev(it)->second;
  a->type = host ? cudaMemoryTypeHost : cudaMemoryTypeDevice;
  a->device = 0;
  a->devicePointer = host ? nullptr : (void *)p;
  a->hostPointer = (void *)p;
  return cudaSuccess;
}

// every page-locked block of the including translation unit is tracked from here on
#define cudaHostAlloc cuemu::host_alloc_tracked
#define cudaFreeHost cuemu::free_host_tracked
