// Shared host-side plumbing of libb200radiomics: error state, CUDA call checking, temporary device buffers, the
// per-device launch state (table blocks, SM count, occupancy, kernel attributes) and the voxel-map kernels' dispatch
// (runtime values to template arguments, launch argument blocks, per-stream scratch).
#pragma once
#include <cuda_runtime.h>
#include <stdio.h>

#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/b200radiomics.h"
#include "host_common.hpp"

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

// ---- voxel-map dispatch: each helper calls f with the type tag of a runtime value and returns f's result
// packed levels: uint8_t or uint16_t
template <typename F>
int with_level_type(int level_bytes, F&& f) {
  if (level_bytes == 1) return f(uint8_t{});
  if (level_bytes == 2) return f(uint16_t{});
  return fail(RB_ERR_ARG, "level_bytes must be 1 or 2");
}
// feature maps: float or double
template <typename F>
int with_map_type(bool out_f32, F&& f) {
  return out_f32 ? f(float{}) : f(double{});
}
// the generic kernels' window class (window_class): std::integral_constant<int, 27 / 125 / 343>
template <typename F>
int with_window_class(int positions, F&& f) {
  switch (window_class(positions)) {
    case 27: return f(std::integral_constant<int, 27>{});
    case 125: return f(std::integral_constant<int, 125>{});
    case GENERIC_WCAP_MAX: return f(std::integral_constant<int, GENERIC_WCAP_MAX>{});
    default: return fail(RB_ERR_UNSUPPORTED, "kernelRadius > 3 is outside the implemented envelope");
  }
}

// The arguments of a texture-class launch (voxel_fast_launch, voxel_features_generic, voxel_features_wide): the packed
// levels, the centres (NULL: every non-zero level), the maps (`out` holds float maps when out_f32, else double;
// feature k of chunk plane z at out + k * fstride + (z - out_z0) * Y * X), the chunk's planes [z0, z1), the word the
// kernels OR their status bits into and the stream every launch runs on.
struct VoxLaunch {
  int cls;
  const void* lev; int level_bytes; const uint8_t* centers; VoxParams P;
  void* out; bool out_f32; long long fstride;
  int z0, z1, out_z0;
  int* status; cudaStream_t st;
};
int voxel_fast_launch(const VoxLaunch& A);
int voxel_features_generic(const VoxLaunch& A);
int voxel_features_wide(const VoxLaunch& A);

// The first-order kernels' parameter block (passed to them by value)
struct FoParams {
  int Z, Y, X;
  long long sz, sy;    // element strides of the (contiguous) image, mask and level volumes
  int rz, ry, rx, z0, z1, out_z0, dtype, level_bytes;
  double shift, voxel_volume, init_value;
};
// The arguments of a first-order launch (firstorder_fast_launch, firstorder_launch, firstorder_wide_launch)
struct FoLaunch {
  const void* img; const uint8_t* mask; const uint8_t* centers; const void* lev;
  FoParams P;
  double* out; long long fstride;
  cudaStream_t st;
};
int firstorder_fast_launch(const FoLaunch& A);
int firstorder_launch(const FoLaunch& A);
int firstorder_wide_launch(const FoLaunch& A);

// ---- per-(device, stream) scratch of the voxel kernels, grown on demand: GLCM's eigen-task queue (tasks, results,
// count, float maps' partial-MCC plane) and the wide kernels' workspace.  A call holds its entry's mutex from taking the
// entry until its last launch on these buffers is enqueued: two host threads on one stream enqueue one after the other
// (in stream order), and a growth or a release never frees a buffer a call is still about to launch on.  Calls on other
// streams never wait for it.  Entries are emptied, never erased (a std::map node does not move), so a pointer to one
// stays valid after the map's own mutex is dropped.
struct ScratchBuf {
  void* p = nullptr;
  size_t bytes = 0;
  template <typename U> U* as() const { return (U*)p; }
};
struct StreamScratch {
  std::mutex mu;
  cudaStream_t st = 0;
  ScratchBuf tasks, results, count, mcc, wide;
  // b holds at least `bytes`: a smaller buffer is freed once the stream has finished with it, then a new one allocated;
  // false, with b empty, if that allocation fails
  bool grow(ScratchBuf& b, size_t bytes) {
    if (b.bytes >= bytes) return true;
    if (b.p) { cudaStreamSynchronize(st); cudaFree(b.p); b.p = nullptr; b.bytes = 0; }
    if (cudaMalloc(&b.p, bytes) != cudaSuccess) { b.p = nullptr; return false; }
    b.bytes = bytes;
    return true;
  }
};
inline std::mutex g_scratch_mu;   // the map only
inline std::map<std::pair<int, cudaStream_t>, StreamScratch> g_scratch;

// the scratch of (current device, st) with its mutex held in lk; nullptr if the device cannot be read
inline StreamScratch* stream_scratch(cudaStream_t st, std::unique_lock<std::mutex>& lk) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  StreamScratch* S;
  {
    std::lock_guard<std::mutex> mlk(g_scratch_mu);
    S = &g_scratch[{dev, st}];
  }
  lk = std::unique_lock<std::mutex>(S->mu);
  S->st = st;
  return S;
}

// rb_release_device_caches: free the current device's scratch (up to 1.15 GB of GLCM queue per stream that ran GLCM,
// up to 1 GiB of wide workspace).  Every entry's mutex is taken first, so no call is between taking its entry and its
// last launch; the device synchronisation then waits for the launches already enqueued.
inline int release_stream_scratch() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return RB_ERR_CUDA;
  std::vector<StreamScratch*> mine;
  {
    std::lock_guard<std::mutex> lk(g_scratch_mu);
    for (auto& kv : g_scratch)
      if (kv.first.first == dev) mine.push_back(&kv.second);
  }
  std::vector<std::unique_lock<std::mutex>> held;
  for (StreamScratch* S : mine) held.emplace_back(S->mu);
  cudaDeviceSynchronize();
  for (StreamScratch* S : mine)
    for (ScratchBuf* b : {&S->tasks, &S->results, &S->count, &S->mcc, &S->wide}) { cudaFree(b->p); *b = ScratchBuf(); }
  return RB_OK;
}

}  // namespace rb
