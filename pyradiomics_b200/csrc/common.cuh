// Shared host-side plumbing of libb200radiomics: error state, CUDA call checking and the per-device launch state
// (table blocks, SM count, occupancy, kernel attributes).
#pragma once
#include <cuda_runtime.h>
#include <stdio.h>

#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <utility>

#include "../../include/b200radiomics.h"

namespace rb {
std::string& last_error_ref();
int fail(int code, const char* fmt, ...);
}  // namespace rb

#define RB_CUDA(call)                                                                          \
  do {                                                                                         \
    cudaError_t _e = (call);                                                                   \
    if (_e != cudaSuccess)                                                                     \
      return rb::fail(_e == cudaErrorMemoryAllocation ? RB_ERR_NOMEM : RB_ERR_CUDA, "%s: %s (%s:%d)", #call, \
                      cudaGetErrorString(_e), __FILE__, __LINE__);                             \
  } while (0)

#define RB_LAUNCH_CHECK() RB_CUDA(cudaGetLastError())

namespace rb {

// A table block built on the host by build(T&) from zeroed memory and copied to the current device once per
// (device, key); it stays for the life of the process.  nullptr if it could not be allocated or copied.
template <typename T, typename Build>
const T* device_table(Build build, int key = 0) {
  static std::mutex mu;
  static std::map<std::pair<int, int>, T*> cache;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find({dev, key});
  if (it != cache.end()) return it->second;
  std::unique_ptr<T> h(new T());
  build(*h);
  T* d = nullptr;
  if (cudaMalloc(&d, sizeof(T)) != cudaSuccess) return nullptr;
  if (cudaMemcpy(d, h.get(), sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(d); return nullptr; }
  return cache[{dev, key}] = d;
}

// SM count of the current device (132 if it cannot be queried)
inline int sm_count() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

// blocks of `block` threads for n items, one item per thread: at most per_sm blocks per SM, at least one block
inline int grid_for(long long n, int block, int per_sm) {
  const long long need = (n + block - 1) / block, cap = (long long)sm_count() * per_sm;
  return (int)(need < cap ? (need < 1 ? 1 : need) : cap);
}

// One block per tile of nt voxels, at most one resident wave (the kernel's occupancy at nt threads and smem bytes of
// dynamic shared memory on every SM, queried once per device): a block that walks many tiles pays its last, partly
// filled tile once.  Set the kernel's dynamic shared-memory limit first.
template <typename K>
cudaError_t resident_grid(K* kernel, int nt, int smem, long long total, int& grid) {
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, int> bps;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  int per_sm = 0;
  {
    std::lock_guard<std::mutex> lk(mu);
    auto it = bps.find({dev, (const void*)kernel});
    if (it != bps.end()) {
      per_sm = it->second;
    } else {
      e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, nt, smem);
      if (e != cudaSuccess) return e;
      bps[{dev, (const void*)kernel}] = per_sm;
    }
  }
  grid = grid_for(total, nt, per_sm > 0 ? per_sm : 1);
  return cudaSuccess;
}

// cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes), once per (device, kernel)
template <typename K>
cudaError_t set_max_dynamic_smem(K* kernel, int bytes) {
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, bool> done;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lk(mu);
  bool& set = done[{dev, (const void*)kernel}];
  if (!set) {
    e = cudaFuncSetAttribute((const void*)kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return e;
    set = true;
  }
  return cudaSuccess;
}

}  // namespace rb
