// Fast fused voxel-based kernels for the headline configuration (kernelRadius 1, 3-D,
// distances [1], 8-bit levels).  One thread per centre voxel, consecutive threads = consecutive
// x so the 24 float64 map stores of a warp are 256-byte coalesced segments.
#include <map>
#include <mutex>

#include "common.cuh"
#define RB_GLCM_BLOCK_SYNC 1   // phase A is called by all threads of a block, uniformly
#include "glcm_fast.cuh"
#include "glcm_kernels.cuh"
#include "glrlm_fast.cuh"
#include "small_fast.cuh"
#include "host_common.hpp"

namespace rb {

bool glcm_fast_applicable(int cls, int level_bytes, const VoxParams& P) {
  return cls == C_GLCM && level_bytes == 1 && P.rz == 1 && P.ry == 1 && P.rx == 1 && P.na == 13 && P.symmetric &&
         !P.weighted && P.Ng <= 255;
}

// per (device, stream) task queue, grown on demand
struct GlcmQueue { GlcmTask* q = nullptr; double* res = nullptr; unsigned* count = nullptr; size_t cap = 0; };
static std::mutex g_queue_mu;
static std::map<std::pair<int, cudaStream_t>, GlcmQueue> g_queue_cache;
// rb_release_device_caches: give the eigen-task queues of the current device back (up to 1.15 GB per stream that ran GLCM)
int glcm_release_queues() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return RB_ERR_CUDA;
  cudaDeviceSynchronize();
  std::lock_guard<std::mutex> lk(g_queue_mu);
  for (auto it = g_queue_cache.begin(); it != g_queue_cache.end();) {
    if (it->first.first == dev) {
      cudaFree(it->second.q); cudaFree(it->second.res); cudaFree(it->second.count);
      it = g_queue_cache.erase(it);
    } else ++it;
  }
  return RB_OK;
}
static GlcmQueue* glcm_queue(cudaStream_t st, size_t need) {
  std::mutex& mu = g_queue_mu;
  auto& cache = g_queue_cache;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  std::lock_guard<std::mutex> lk(mu);
  GlcmQueue& Q = cache[{dev, st}];
  if (!Q.count && cudaMalloc(&Q.count, sizeof(unsigned)) != cudaSuccess) return nullptr;
  if (Q.cap < need) {
    if (Q.q) { cudaStreamSynchronize(st); cudaFree(Q.q); cudaFree(Q.res); Q.q = nullptr; Q.res = nullptr; Q.cap = 0; }
    if (cudaMalloc(&Q.q, need * sizeof(GlcmTask)) != cudaSuccess) return nullptr;
    if (cudaMalloc(&Q.res, need * sizeof(double)) != cudaSuccess) { cudaFree(Q.q); Q.q = nullptr; return nullptr; }
    Q.cap = need;
  }
  return &Q;
}

int glcm_fast_launch(const void* lev, const uint8_t* centers, const VoxParams& P, double* out, long long fstride,
                     int z0, int z1, int out_z0, cudaStream_t st) {
  const GlcmFastTables* T = device_table<GlcmFastTables>([&](GlcmFastTables& h) { glcm_fast_build_tables(h, P.Ng); }, P.Ng);
  if (!T) return fail(RB_ERR_CUDA, "could not build the GLCM table block on the device");
  const long long plane = (long long)P.Y * P.X;
  if ((long long)(z1 - z0) * plane <= 0) return RB_OK;
  if (P.sy != P.X || P.sz != plane) return fail(RB_ERR_ARG, "GLCM fast path expects a contiguous level volume");
  const int sms = sm_count();
  // chunk of planes whose worst-case queue (13 eigen-tasks per voxel) stays <= 48 Mi entries
  // (768 MB of tasks + 384 MB of results)
  const long long max_entries = 48ll << 20;
  int zchunk = (int)(max_entries / (plane * GF_NA));
  if (zchunk < 1) zchunk = 1;
  if (zchunk > z1 - z0) zchunk = z1 - z0;
  GlcmQueue* Q = glcm_queue(st, (size_t)zchunk * plane * GF_NA);
  if (!Q) return fail(RB_ERR_NOMEM, "could not allocate the GLCM eigen-task queue");
  // phase A: one CTA per SM (register-bound).  512 threads at 128 registers (a hundred spilled words per thread, L1-
  // resident) put 16 warps on an SM instead of the 8 of a 256-thread / 236-register build, which hides more of the
  // latency of this issue-bound kernel.
  constexpr int NT = 512;
  const int smem = glcm_phaseA_smem_bytes(NT);
  RB_CUDA(set_max_dynamic_smem(glcm_fast_kernel<1, NT>, smem));
  // register Lanczos: 90 KB of per-thread shared vectors per CTA -> two CTAs per SM
  RB_CUDA(set_max_dynamic_smem(glcm_fast_solve_kernel<2>, GF_LZ_SMEM_BYTES));
  const uint8_t* l8 = (const uint8_t*)lev;
  for (int za = z0; za < z1; za += zchunk) {
    const int zb = za + zchunk < z1 ? za + zchunk : z1;
    RB_CUDA(cudaMemsetAsync(Q->count, 0, sizeof(unsigned), st));
    int grid = 0;
    RB_CUDA(resident_grid(glcm_fast_kernel<1, NT>, NT, smem, (long long)(zb - za) * plane, grid));
    glcm_fast_kernel<1, NT><<<grid, NT, smem, st>>>(l8, centers, P, T, out, fstride, za, zb, out_z0, Q->q, Q->count);
    RB_LAUNCH_CHECK();
    // One launch per size group keeps ONE solver body in the instruction cache (the three Lanczos templates together are
    // 18.5 k SASS instructions, 296 KB, and on a smooth volume the blocks of an SM otherwise sit in different groups); the
    // dense n <= 8 solves stay a single launch, where the repeated tile sorts would cost more than they save.
    glcm_fast_solve_kernel<0><<<sms * 8, 128, 0, st>>>(l8, P, T, Q->q, Q->count, Q->res, 0);
    for (int g = 10; g <= 12; g += 2) glcm_fast_solve_kernel<1><<<sms * 8, 128, 0, st>>>(l8, P, T, Q->q, Q->count, Q->res, g);
    for (int g = 18; g >= 14; g -= 2)
      glcm_fast_solve_kernel<2><<<sms * 2, 128, GF_LZ_SMEM_BYTES, st>>>(l8, P, T, Q->q, Q->count, Q->res, g);
    RB_LAUNCH_CHECK();
    glcm_fast_finish_kernel<<<sms * 8, 256, 0, st>>>(P, Q->q, Q->count, Q->res, out + (long long)G_MCC * fstride, out_z0);
    RB_LAUNCH_CHECK();
  }
  return RB_OK;
}

// ---------------------------------------------------------------------------------- GLRLM
__global__ void __launch_bounds__(128)
glrlm_fast_kernel(const uint8_t* __restrict__ lev, const uint8_t* __restrict__ centers,
                  const __grid_constant__ VoxParams P, const GlrlmFastTables* __restrict__ Tg,
                  double* __restrict__ out, long long fstride, int z0, int z1, int out_z0) {
  __shared__ GlrlmFastTables T;
  copy_tables_to_shared(T, Tg);
  __syncthreads();
  const long long plane = (long long)P.Y * P.X;
  const long long total = (long long)(z1 - z0) * plane;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const ChunkVoxel v = chunk_voxel(P, plane, z0, out_z0, t);
    if (!chunk_center(lev, centers, plane, v)) {
#pragma unroll
      for (int k = 0; k < GLRLM_NF; k++) out[k * fstride + v.oi] = P.init_value;
      continue;
    }
    int wl[27];
    load_window27(lev, P, v.z, v.y, v.x, v.vi, true, wl, 1);
    double f[GLRLM_NF];
    glrlm_fast_voxel(wl, T, f);
#pragma unroll
    for (int k = 0; k < GLRLM_NF; k++) out[k * fstride + v.oi] = f[k];
  }
}

bool glrlm_fast_applicable(int cls, int level_bytes, const VoxParams& P) {
  return cls == C_GLRLM && level_bytes == 1 && P.rz == 1 && P.ry == 1 && P.rx == 1 && P.na == 13 && !P.weighted && P.Ng <= 255;
}

int glrlm_fast_launch(const void* lev, const uint8_t* centers, const VoxParams& P, double* out, long long fstride,
                      int z0, int z1, int out_z0, cudaStream_t st) {
  const GlrlmFastTables* T = device_table<GlrlmFastTables>(glrlm_fast_build_tables);
  if (!T) return fail(RB_ERR_CUDA, "could not build the GLRLM table block on the device");
  const long long total = (long long)(z1 - z0) * P.Y * P.X;
  if (total <= 0) return RB_OK;
  glrlm_fast_kernel<<<grid_for(total, 128, 32), 128, 0, st>>>((const uint8_t*)lev, centers, P, T, out, fstride, z0, z1, out_z0);
  RB_LAUNCH_CHECK();
  return RB_OK;
}

// ------------------------------------------------------------------ GLSZM / GLDM / NGTDM fast paths
// SYNC: block-uniform tiles with a barrier per tile, so the block's warps stream the (large,
// straight-line) GLDM body together and share instruction-cache lines (free-running warps stall
// on instruction fetch).
template <int CLS, int NT, bool SYNC>
__global__ void __launch_bounds__(NT)
small_fast_kernel(const uint8_t* __restrict__ lev, const uint8_t* __restrict__ centers,
                  const __grid_constant__ VoxParams P, const SmallFastTables* __restrict__ Tg,
                  double* __restrict__ out, long long fstride, int z0, int z1, int out_z0) {
  __shared__ SmallFastTables T;
  copy_tables_to_shared<NT>(T, Tg);
  __syncthreads();
  constexpr int NF = CLS == C_GLSZM ? GLSZM_NF : GLDM_NF;
  const long long plane = (long long)P.Y * P.X;
  const long long total = (long long)(z1 - z0) * plane;
  const long long ntiles = (total + NT - 1) / NT;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    if (SYNC) __syncthreads();
    const long long t = tile * NT + threadIdx.x;
    const bool live = t < total;
    if (!SYNC && !live) continue;
    const ChunkVoxel v = chunk_voxel(P, plane, z0, out_z0, t, live);
    const bool is_center = live && chunk_center(lev, centers, plane, v);
    if (!SYNC && !is_center) {
#pragma unroll
      for (int k = 0; k < NF; k++) out[k * fstride + v.oi] = P.init_value;
      continue;
    }
    int wl[27];
    load_window27(lev, P, v.z, v.y, v.x, v.vi, is_center, wl, 1);
    double f[16];
    if (CLS == C_GLSZM) glszm_fast_voxel(wl, T, f);
    else gldm_fast_voxel(wl, P.alpha, T, f);
    if (!live) continue;
#pragma unroll
    for (int k = 0; k < NF; k++) out[k * fstride + v.oi] = is_center ? f[k] : P.init_value;
  }
}

// NGTDM over the full/deferred tiles of full_window_tiles (voxel_tiles.cuh).  Per-thread scratch for the level classes
// lives in shared memory, [entry][thread].
constexpr int NGTDM_NT = 128;
template <int NT>
__global__ void __launch_bounds__(NT, 4)
ngtdm_fast_kernel(const uint8_t* __restrict__ lev, const uint8_t* __restrict__ centers,
                  const __grid_constant__ VoxParams P, const SmallFastTables* __restrict__ Tg,
                  double* __restrict__ out, long long fstride, int z0, int z1, int out_z0) {
  __shared__ SmallFastTables T;
  __shared__ double ng_ns[27 * NT];
  __shared__ int ng_pk[27 * NT];
  __shared__ long long defer[2 * NT];                              // chunk indices of the centres left to the general body
  __shared__ unsigned ndefer;
  copy_tables_to_shared<NT>(T, Tg);
  const int tid = threadIdx.x;
  if (tid == 0) ndefer = 0;
  __syncthreads();
  const long long plane = (long long)P.Y * P.X;
  full_window_tiles<NT>((long long)(z1 - z0) * plane, defer, ndefer,
    [&](long long t, bool live, auto defer_it) {
      if (!live) return;
      const ChunkVoxel v = chunk_voxel(P, plane, z0, out_z0, t);
      const bool is_center = chunk_center(lev, centers, plane, v);
      int wl[27];
      load_window27(lev, P, v.z, v.y, v.x, v.vi, is_center, wl, 1);
      if (is_center && ngtdm_window_full(wl)) {
        double f[NGTDM_NF];
        ngtdm_fast_body<true>(wl, T, f, ng_pk + tid, ng_ns + tid, NT);
#pragma unroll
        for (int k = 0; k < NGTDM_NF; k++) out[k * fstride + v.oi] = f[k];
      } else if (is_center) {
        defer_it();
      } else {
#pragma unroll
        for (int k = 0; k < NGTDM_NF; k++) out[k * fstride + v.oi] = P.init_value;
      }
    },
    [&](auto entry, bool live) {
      if (!live) return;
      const ChunkVoxel v = chunk_voxel(P, plane, z0, out_z0, entry());
      const bool is_center = chunk_center(lev, centers, plane, v);
      int wl[27];
      load_window27(lev, P, v.z, v.y, v.x, v.vi, is_center, wl, 1);
      double f[NGTDM_NF];
      ngtdm_fast_body<false>(wl, T, f, ng_pk + tid, ng_ns + tid, NT);
#pragma unroll
      for (int k = 0; k < NGTDM_NF; k++) out[k * fstride + v.oi] = f[k];
    });
}

bool small_fast_applicable(int cls, int level_bytes, const VoxParams& P) {
  return (cls == C_GLSZM || cls == C_GLDM || cls == C_NGTDM) && level_bytes == 1 && P.rz == 1 && P.ry == 1 && P.rx == 1 &&
         P.na == 26 && P.Ng <= 255;
}

int small_fast_launch(int cls, const void* lev, const uint8_t* centers, const VoxParams& P, double* out, long long fstride,
                      int z0, int z1, int out_z0, cudaStream_t st) {
  const SmallFastTables* T = device_table<SmallFastTables>(small_fast_build_tables);
  if (!T) return fail(RB_ERR_CUDA, "could not build the table block on the device");
  const long long total = (long long)(z1 - z0) * P.Y * P.X;
  if (total <= 0) return RB_OK;
  const uint8_t* l8 = (const uint8_t*)lev;
  if (cls == C_NGTDM) {
    int grid = 0;
    RB_CUDA(resident_grid(ngtdm_fast_kernel<NGTDM_NT>, NGTDM_NT, 0, total, grid));
    ngtdm_fast_kernel<NGTDM_NT><<<grid, NGTDM_NT, 0, st>>>(l8, centers, P, T, out, fstride, z0, z1, out_z0);
  } else if (cls == C_GLSZM) {
    small_fast_kernel<C_GLSZM, 128, false><<<grid_for(total, 128, 32), 128, 0, st>>>(l8, centers, P, T, out, fstride, z0, z1, out_z0);
  } else {
    small_fast_kernel<C_GLDM, 256, true><<<grid_for(total, 256, 16), 256, 0, st>>>(l8, centers, P, T, out, fstride, z0, z1, out_z0);
  }
  RB_LAUNCH_CHECK();
  return RB_OK;
}

}  // namespace rb
