// Fast fused voxel-based kernels for the headline configuration (kernelRadius 1, 3-D,
// distances [1], 8-bit levels).  One thread per centre voxel, consecutive threads = consecutive
// x so the 24 float64 map stores of a warp are 256-byte coalesced segments.
#include <stdlib.h>

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

#ifndef GF_SOLVE_SPLIT
#define GF_SOLVE_SPLIT 3
#endif
#ifndef GF_PHASEA_NT
#define GF_PHASEA_NT 512
#endif



// device-resident table cache, one per (device, Ng)
static const GlcmFastTables* glcm_fast_tables_dev(int Ng) {
  static std::mutex mu;
  static std::map<std::pair<int, int>, GlcmFastTables*> cache;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find({dev, Ng});
  if (it != cache.end()) return it->second;
  GlcmFastTables* h = new GlcmFastTables;
  memset(h, 0, sizeof *h);
  glcm_fast_build_tables(*h, Ng);
  GlcmFastTables* d = nullptr;
  if (cudaMalloc(&d, sizeof *h) != cudaSuccess || cudaMemcpy(d, h, sizeof *h, cudaMemcpyHostToDevice) != cudaSuccess) {
    delete h;
    return nullptr;
  }
  delete h;
  cache[{dev, Ng}] = d;
  return d;
}

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
  const GlcmFastTables* T = glcm_fast_tables_dev(P.Ng);
  if (!T) return fail(RB_ERR_CUDA, "could not build the GLCM table block on the device");
  const long long plane = (long long)P.Y * P.X;
  if ((long long)(z1 - z0) * plane <= 0) return RB_OK;
  if (P.sy != P.X || P.sz != plane) return fail(RB_ERR_ARG, "GLCM fast path expects a contiguous level volume");
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  // chunk of planes whose worst-case queue (13 eigen-tasks per voxel) stays <= 48 Mi entries
  // (768 MB of tasks + 384 MB of results)
  const long long max_entries = 48ll << 20;
  int zchunk = (int)(max_entries / (plane * GF_NA));
  if (zchunk < 1) zchunk = 1;
  if (zchunk > z1 - z0) zchunk = z1 - z0;
  GlcmQueue* Q = glcm_queue(st, (size_t)zchunk * plane * GF_NA);
  if (!Q) return fail(RB_ERR_NOMEM, "could not allocate the GLCM eigen-task queue");
  for (int za = z0; za < z1; za += zchunk) {
    const int zb = za + zchunk < z1 ? za + zchunk : z1;
    const long long total = (long long)(zb - za) * plane;
    RB_CUDA(cudaMemsetAsync(Q->count, 0, sizeof(unsigned), st));
    // phase A: one CTA per SM (register-bound).  512 threads at 128 registers (a hundred spilled words per thread, L1-
    // resident) put 16 warps on an SM instead of the 8 of the 256-thread / 236-register build, which hides more of the
    // latency of this issue-bound kernel; 384 threads sit in between.  B200_GLCM_NT selects the variant for A/B runs.
    static const int nt = getenv("B200_GLCM_NT") ? atoi(getenv("B200_GLCM_NT")) : GF_PHASEA_NT;
    const uint8_t* l8 = (const uint8_t*)lev;
    static bool pa_attr[64] = {false};
    static int pa_bps[64][3];
    if (!pa_attr[dev & 63]) {
      RB_CUDA(cudaFuncSetAttribute(glcm_fast_kernel<1, 256>, cudaFuncAttributeMaxDynamicSharedMemorySize, glcm_phaseA_smem_bytes(256)));
      RB_CUDA(cudaFuncSetAttribute(glcm_fast_kernel<1, 384>, cudaFuncAttributeMaxDynamicSharedMemorySize, glcm_phaseA_smem_bytes(384)));
      RB_CUDA(cudaFuncSetAttribute(glcm_fast_kernel<1, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, glcm_phaseA_smem_bytes(512)));
      RB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&pa_bps[dev & 63][0], glcm_fast_kernel<1, 256>, 256, glcm_phaseA_smem_bytes(256)));
      RB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&pa_bps[dev & 63][1], glcm_fast_kernel<1, 384>, 384, glcm_phaseA_smem_bytes(384)));
      RB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&pa_bps[dev & 63][2], glcm_fast_kernel<1, 512>, 512, glcm_phaseA_smem_bytes(512)));
      pa_attr[dev & 63] = true;
    }
    // one resident wave of blocks, each walking many tiles: a block runs its list of non-full windows in whole tiles,
    // so its last, partly filled tile is paid once per block rather than once per short-lived block
    const int bps = pa_bps[dev & 63][nt == 512 ? 2 : nt == 384 ? 1 : 0];
    const long long need = (total + nt - 1) / nt, cap = (long long)sms * (bps > 0 ? bps : 1);
    const int grid = (int)(need < cap ? need : cap);
    if (nt == 512) glcm_fast_kernel<1, 512><<<grid, 512, glcm_phaseA_smem_bytes(512), st>>>(l8, centers, P, T, out, fstride, za, zb, out_z0, Q->q, Q->count);
    else if (nt == 384) glcm_fast_kernel<1, 384><<<grid, 384, glcm_phaseA_smem_bytes(384), st>>>(l8, centers, P, T, out, fstride, za, zb, out_z0, Q->q, Q->count);
    else glcm_fast_kernel<1, 256><<<grid, 256, glcm_phaseA_smem_bytes(256), st>>>(l8, centers, P, T, out, fstride, za, zb, out_z0, Q->q, Q->count);
    RB_LAUNCH_CHECK();
    static const int solve_bps = getenv("B200_GLCM_SOLVE_BPS") ? atoi(getenv("B200_GLCM_SOLVE_BPS")) : 8;
    // One launch per size group keeps ONE solver body in the instruction cache (the three Lanczos templates together are
    // 18.5 k SASS instructions, 296 KB, and on a smooth volume the blocks of an SM otherwise sit in different groups); the
    // dense n <= 8 solves stay a single launch, where the repeated tile sorts would cost more than they save.
    // B200_GLCM_SPLIT: bit 0 Lanczos, bit 1 dense <= 12, bit 2 dense <= 8 (A/B switch).
    static const int split = getenv("B200_GLCM_SPLIT") ? atoi(getenv("B200_GLCM_SPLIT")) : GF_SOLVE_SPLIT;
    if (split & 4) {
      for (int g = 4; g <= 8; g += 2) glcm_fast_solve_kernel<0><<<sms * solve_bps, 128, 0, st>>>((const uint8_t*)lev, P, T, Q->q, Q->count, Q->res, g);
    } else {
      glcm_fast_solve_kernel<0><<<sms * solve_bps, 128, 0, st>>>((const uint8_t*)lev, P, T, Q->q, Q->count, Q->res, 0);
    }
    if (split & 2) {
      for (int g = 10; g <= 12; g += 2) glcm_fast_solve_kernel<1><<<sms * solve_bps, 128, 0, st>>>((const uint8_t*)lev, P, T, Q->q, Q->count, Q->res, g);
    } else {
      glcm_fast_solve_kernel<1><<<sms * solve_bps, 128, 0, st>>>((const uint8_t*)lev, P, T, Q->q, Q->count, Q->res, 0);
    }
    // register Lanczos: 90 KB of per-thread shared vectors per CTA -> two CTAs per SM
    static bool lz_attr[64] = {false};
    if (!lz_attr[dev & 63]) {
      RB_CUDA(cudaFuncSetAttribute(glcm_fast_solve_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, GF_LZ_SMEM_BYTES));
      lz_attr[dev & 63] = true;
    }
    if (split & 1) {
      for (int g = 18; g >= 14; g -= 2) glcm_fast_solve_kernel<2><<<sms * 2, 128, GF_LZ_SMEM_BYTES, st>>>((const uint8_t*)lev, P, T, Q->q, Q->count, Q->res, g);
    } else {
      glcm_fast_solve_kernel<2><<<sms * 2, 128, GF_LZ_SMEM_BYTES, st>>>((const uint8_t*)lev, P, T, Q->q, Q->count, Q->res, 0);
    }
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
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(Tg);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&T);
    for (int i = threadIdx.x; i < (int)(sizeof(GlrlmFastTables) / 4); i += blockDim.x) dst[i] = src[i];
  }
  __syncthreads();
  const long long plane = (long long)P.Y * P.X;
  const long long total = (long long)(z1 - z0) * plane;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int z = z0 + (int)(t / plane);
    const int rem = (int)(t % plane);
    const int y = rem / P.X, x = rem % P.X;
    const long long vi = (long long)z * P.sz + (long long)y * P.sy + x;
    const long long oi = (long long)(z - out_z0) * plane + rem;
    const bool is_center = centers ? centers[(long long)z * plane + rem] != 0 : lev[vi] != 0;
    if (!is_center) {
#pragma unroll
      for (int k = 0; k < GLRLM_NF; k++) out[k * fstride + oi] = P.init_value;
      continue;
    }
    int wl[27];
    {
      int p = 0;
#pragma unroll
      for (int dz = -1; dz <= 1; dz++)
#pragma unroll
        for (int dy = -1; dy <= 1; dy++)
#pragma unroll
          for (int dx = -1; dx <= 1; dx++, p++) {
            const int zz = z + dz, yy = y + dy, xx = x + dx;
            const bool in = zz >= 0 && zz < P.Z && yy >= 0 && yy < P.Y && xx >= 0 && xx < P.X;
            wl[p] = in ? lev[vi + (long long)dz * P.sz + (long long)dy * P.sy + dx] : 0;
          }
    }
    double f[GLRLM_NF];
    glrlm_fast_voxel(wl, T, f);
#pragma unroll
    for (int k = 0; k < GLRLM_NF; k++) out[k * fstride + oi] = f[k];
  }
}

static const GlrlmFastTables* glrlm_fast_tables_dev() {
  static std::mutex mu;
  static std::map<int, GlrlmFastTables*> cache;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(dev);
  if (it != cache.end()) return it->second;
  GlrlmFastTables* h = new GlrlmFastTables;
  memset(h, 0, sizeof *h);
  glrlm_fast_build_tables(*h);
  GlrlmFastTables* d = nullptr;
  if (cudaMalloc(&d, sizeof *h) != cudaSuccess || cudaMemcpy(d, h, sizeof *h, cudaMemcpyHostToDevice) != cudaSuccess) { delete h; return nullptr; }
  delete h;
  cache[dev] = d;
  return d;
}

bool glrlm_fast_applicable(int cls, int level_bytes, const VoxParams& P) {
  return cls == C_GLRLM && level_bytes == 1 && P.rz == 1 && P.ry == 1 && P.rx == 1 && P.na == 13 && !P.weighted && P.Ng <= 255;
}

int glrlm_fast_launch(const void* lev, const uint8_t* centers, const VoxParams& P, double* out, long long fstride,
                      int z0, int z1, int out_z0, cudaStream_t st) {
  const GlrlmFastTables* T = glrlm_fast_tables_dev();
  if (!T) return fail(RB_ERR_CUDA, "could not build the GLRLM table block on the device");
  const long long total = (long long)(z1 - z0) * P.Y * P.X;
  if (total <= 0) return RB_OK;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  long long need = (total + 127) / 128, cap = (long long)sms * 32;
  glrlm_fast_kernel<<<(int)(need < cap ? need : cap), 128, 0, st>>>((const uint8_t*)lev, centers, P, T, out, fstride, z0, z1, out_z0);
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
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(Tg);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&T);
    for (int i = threadIdx.x; i < (int)(sizeof(SmallFastTables) / 4); i += NT) dst[i] = src[i];
  }
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
    const int z = z0 + (int)((live ? t : 0) / plane);
    const int rem = (int)((live ? t : 0) % plane);
    const int y = rem / P.X, x = rem % P.X;
    const long long vi = (long long)z * P.sz + (long long)y * P.sy + x;
    const long long oi = (long long)(z - out_z0) * plane + rem;
    const bool is_center = live && (centers ? centers[(long long)z * plane + rem] != 0 : lev[vi] != 0);
    if (!SYNC && !is_center) {
#pragma unroll
      for (int k = 0; k < NF; k++) out[k * fstride + oi] = P.init_value;
      continue;
    }
    int wl[27];
    {
      int p = 0;
#pragma unroll
      for (int dz = -1; dz <= 1; dz++)
#pragma unroll
        for (int dy = -1; dy <= 1; dy++)
#pragma unroll
          for (int dx = -1; dx <= 1; dx++, p++) {
            const int zz = z + dz, yy = y + dy, xx = x + dx;
            const bool in = is_center && zz >= 0 && zz < P.Z && yy >= 0 && yy < P.Y && xx >= 0 && xx < P.X;
            wl[p] = in ? lev[vi + (long long)dz * P.sz + (long long)dy * P.sy + dx] : 0;
          }
    }
    double f[16];
    if (CLS == C_GLSZM) glszm_fast_voxel(wl, T, f);
    else gldm_fast_voxel(wl, P.alpha, T, f);
    if (!live) continue;
#pragma unroll
    for (int k = 0; k < NF; k++) out[k * fstride + oi] = is_center ? f[k] : P.init_value;
  }
}

// NGTDM: block-uniform tiles of NT voxels.  A centre with a full window runs the full-window body at once, a voxel that
// is not a centre stores init_value, and any other centre (the volume's faces, the ROI's border and holes) goes to the
// block's list, which the block runs through the general body NT at a time whenever NT are waiting, and once at the end
// (the scheme of GLCM phase A: no warp runs both bodies for one tile).  Per-thread scratch for the level classes lives
// in shared memory, [entry][thread].
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
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(Tg);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&T);
    for (int i = threadIdx.x; i < (int)(sizeof(SmallFastTables) / 4); i += NT) dst[i] = src[i];
  }
  const int tid = threadIdx.x;
  if (tid == 0) ndefer = 0;
  __syncthreads();
  const long long plane = (long long)P.Y * P.X;
  const long long total = (long long)(z1 - z0) * plane;
  const long long ntiles = (total + NT - 1) / NT;
  // voxel t of the chunk: its window (zeros outside the volume), output index and whether it is a centre
  auto load = [&](long long t, int* wl, long long& oi) -> bool {
    const int z = z0 + (int)(t / plane);
    const int rem = (int)(t % plane);
    const int y = rem / P.X, x = rem % P.X;
    const long long vi = (long long)z * P.sz + (long long)y * P.sy + x;
    oi = (long long)(z - out_z0) * plane + rem;
    const bool is_center = centers ? centers[(long long)z * plane + rem] != 0 : lev[vi] != 0;
    int p = 0;
#pragma unroll
    for (int dz = -1; dz <= 1; dz++)
#pragma unroll
      for (int dy = -1; dy <= 1; dy++)
#pragma unroll
        for (int dx = -1; dx <= 1; dx++, p++) {
          const int zz = z + dz, yy = y + dy, xx = x + dx;
          const bool in = is_center && zz >= 0 && zz < P.Z && yy >= 0 && yy < P.Y && xx >= 0 && xx < P.X;
          wl[p] = in ? lev[vi + (long long)dz * P.sz + (long long)dy * P.sy + dx] : 0;
        }
    return is_center;
  };
  // one pass per tile and a last pass with no tile (one call site per body)
  for (long long tile = blockIdx.x;; tile += gridDim.x) {
    const bool more = tile < ntiles;                                 // block-uniform
    if (more) {
      const long long t = tile * NT + tid;
      if (t < total) {
        int wl[27];
        long long oi;
        const bool is_center = load(t, wl, oi);
        if (is_center && ngtdm_window_full(wl)) {
          double f[NGTDM_NF];
          ngtdm_fast_body<true>(wl, T, f, ng_pk + tid, ng_ns + tid, NT);
#pragma unroll
          for (int k = 0; k < NGTDM_NF; k++) out[k * fstride + oi] = f[k];
        } else if (is_center) {
          defer[atomicAdd(&ndefer, 1u)] = t;
        } else {
#pragma unroll
          for (int k = 0; k < NGTDM_NF; k++) out[k * fstride + oi] = P.init_value;
        }
      }
    }
    __syncthreads();
    const unsigned nd = ndefer;
    __syncthreads();
    // the general body over the last `count` list entries
    const unsigned count = more ? (nd >= NT ? NT : 0) : nd;
    if (count) {
      if (tid == 0) ndefer = nd - count;
      if ((unsigned)tid < count) {
        int wl[27];
        long long oi;
        load(defer[nd - count + tid], wl, oi);
        double f[NGTDM_NF];
        ngtdm_fast_body<false>(wl, T, f, ng_pk + tid, ng_ns + tid, NT);
#pragma unroll
        for (int k = 0; k < NGTDM_NF; k++) out[k * fstride + oi] = f[k];
      }
      __syncthreads();                                               // every entry read before the list grows again
    }
    if (!more) break;
  }
}

static const SmallFastTables* small_fast_tables_dev() {
  static std::mutex mu;
  static std::map<int, SmallFastTables*> cache;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(dev);
  if (it != cache.end()) return it->second;
  SmallFastTables* h = new SmallFastTables;
  small_fast_build_tables(*h);
  SmallFastTables* d = nullptr;
  if (cudaMalloc(&d, sizeof *h) != cudaSuccess || cudaMemcpy(d, h, sizeof *h, cudaMemcpyHostToDevice) != cudaSuccess) { delete h; return nullptr; }
  delete h;
  cache[dev] = d;
  return d;
}

bool small_fast_applicable(int cls, int level_bytes, const VoxParams& P) {
  return (cls == C_GLSZM || cls == C_GLDM || cls == C_NGTDM) && level_bytes == 1 && P.rz == 1 && P.ry == 1 && P.rx == 1 &&
         P.na == 26 && P.Ng <= 255;
}

int small_fast_launch(int cls, const void* lev, const uint8_t* centers, const VoxParams& P, double* out, long long fstride,
                      int z0, int z1, int out_z0, cudaStream_t st) {
  const SmallFastTables* T = small_fast_tables_dev();
  if (!T) return fail(RB_ERR_CUDA, "could not build the table block on the device");
  const long long total = (long long)(z1 - z0) * P.Y * P.X;
  if (total <= 0) return RB_OK;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const uint8_t* l8 = (const uint8_t*)lev;
  if (cls == C_NGTDM) {
    // one resident wave of blocks, each walking many tiles: a block's last, partly filled list tile is paid once
    static int ng_bps[64] = {0};
    if (!ng_bps[dev & 63]) RB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ng_bps[dev & 63], ngtdm_fast_kernel<NGTDM_NT>, NGTDM_NT, 0));
    const long long need = (total + NGTDM_NT - 1) / NGTDM_NT, cap = (long long)sms * (ng_bps[dev & 63] > 0 ? ng_bps[dev & 63] : 1);
    ngtdm_fast_kernel<NGTDM_NT><<<(int)(need < cap ? need : cap), NGTDM_NT, 0, st>>>(l8, centers, P, T, out, fstride, z0, z1, out_z0);
    RB_LAUNCH_CHECK();
    return RB_OK;
  }
  static const int mode_env = getenv("B200_SMALL_MODE") ? atoi(getenv("B200_SMALL_MODE")) : -1;   // GLDM: 0 free-running, 1 sync/128, 2 sync/256, -1: measured best
  const int mode = mode_env >= 0 ? mode_env : 2;
  if (cls == C_GLSZM || mode == 0) {
    long long need = (total + 127) / 128, cap = (long long)sms * 32;
    const int grid = (int)(need < cap ? need : cap);
    if (cls == C_GLSZM) small_fast_kernel<C_GLSZM, 128, false><<<grid, 128, 0, st>>>(l8, centers, P, T, out, fstride, z0, z1, out_z0);
    else small_fast_kernel<C_GLDM, 128, false><<<grid, 128, 0, st>>>(l8, centers, P, T, out, fstride, z0, z1, out_z0);
  } else if (mode == 1) {
    long long need = (total + 127) / 128, cap = (long long)sms * 32;
    const int grid = (int)(need < cap ? need : cap);
    small_fast_kernel<C_GLDM, 128, true><<<grid, 128, 0, st>>>(l8, centers, P, T, out, fstride, z0, z1, out_z0);
  } else {
    long long need = (total + 255) / 256, cap = (long long)sms * 16;
    const int grid = (int)(need < cap ? need : cap);
    small_fast_kernel<C_GLDM, 256, true><<<grid, 256, 0, st>>>(l8, centers, P, T, out, fstride, z0, z1, out_z0);
  }
  RB_LAUNCH_CHECK();
  return RB_OK;
}

}  // namespace rb
