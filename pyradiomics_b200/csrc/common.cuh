// Shared host-side plumbing of libb200radiomics: error state, CUDA call checking, temporary device buffers and the
// per-device launch state (table blocks, SM count, occupancy, kernel attributes).
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
// The copy has landed before the pointer is handed out: a plain cudaMemcpy from pageable memory may return while its
// DMA is still in flight, ordered only with the legacy default stream, and the caller launches on its own (possibly
// non-blocking) stream.  So it runs on a private stream that is synchronised, which stalls no other stream.
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
  cudaStream_t s = nullptr;
  if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess) { cudaFree(d); return nullptr; }
  const bool ok = cudaMemcpyAsync(d, h.get(), sizeof(T), cudaMemcpyHostToDevice, s) == cudaSuccess &&
                  cudaStreamSynchronize(s) == cudaSuccess;
  cudaStreamDestroy(s);
  if (!ok) { cudaFree(d); return nullptr; }
  return cache[{dev, key}] = d;
}

// One temporary device buffer, freed (cudaFree, synchronous) when it goes out of scope.  Wrap alloc in RB_CUDA so an
// allocation failure reports RB_ERR_NOMEM.
struct DevBuf {
  void* p = nullptr;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { if (p) cudaFree(p); }
  cudaError_t alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 1); }
  template <typename U> U* as() const { return (U*)p; }
};

// The opaque handle between GLSZM's two phases: the zones as (gray, size) int pairs, and the stream phase one ran on,
// where the fill (matrix_kernels.cu glszm_fill) runs too.
struct GlszmHandle {
  bool batch = false;
  cudaStream_t st = 0;
  int nvox = 1, wcap = 0;
  unsigned nzones = 0;
  DevBuf zones;   // segment: int[2*nzones]; batch: int[nvox][2*wcap]
  DevBuf nz;      // batch: int[nvox]
};

// Segment-mode builders (segment_kernels.cu): one ROI's matrices from packed levels (uint8 or uint16, size[nd], nd = 2
// or 3) into HOST float64 buffers, or GLSZM's zones into a new handle; every launch and copy runs on `st`.
int segment_matrices(const void* lev, int level_bytes, const int* size, int nd, const int* distances, int ndist, int Ng,
                     int alpha, int force2D, int force2Ddimension, double* glcm_host, double* gldm_host, double* ngtdm_host,
                     int* angles_out, cudaStream_t st);
int segment_glrlm(const void* lev, int level_bytes, const int* size, int nd, int Ng, int Nr, int force2D, int force2Ddimension,
                  double* glrlm_host, int* angles_out, cudaStream_t st);
int segment_glszm(const void* lev, int level_bytes, const int* size, int nd, int Ng, int force2D, int force2Ddimension,
                  int* max_region, void** handle, cudaStream_t st);

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
