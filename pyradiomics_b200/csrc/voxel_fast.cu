// Fast fused voxel-based kernels for the headline configuration (kernelRadius 1, 3-D,
// distances [1], 8-bit levels).  One thread per centre voxel, consecutive threads = consecutive
// x so the 24 float64 map stores of a warp are 256-byte coalesced segments (128-byte for float32 maps).
// Every kernel and launch function takes the map type (double or float, store_map in voxel_tiles.cuh).
#include "common.cuh"
#define RB_GLCM_BLOCK_SYNC 1   // phase A is called by all threads of a block, uniformly
#include "glcm_fast.cuh"
#include "glcm_kernels.cuh"
#include "glrlm_fast.cuh"
#include "small_fast.cuh"

namespace rb {

template <typename OutT>
static int glcm_fast_run(const uint8_t* l8, const uint8_t* centers, const VoxParams& P, OutT* out, long long fstride,
                         int z0, int z1, int out_z0, cudaStream_t st) {
  const GlcmFastTables* T = device_table<GlcmFastTables>([&](GlcmFastTables& h) { glcm_fast_build_tables(h, P.Ng); }, P.Ng);
  if (!T) return fail(RB_ERR_CUDA, "could not build the GLCM table block on the device");
  const long long plane = (long long)P.Y * P.X;
  if ((long long)(z1 - z0) * plane <= 0) return RB_OK;
  if (P.sy != P.X || P.sz != plane) return fail(RB_ERR_ARG, "GLCM fast path expects a contiguous level volume");
  const int sms = sm_count();
  // chunk of planes whose worst-case queue (13 eigen-tasks per voxel) stays <= 48 Mi entries
  // (768 MB of tasks + 384 MB of results); the planes are spread evenly over the chunks, so the last one is not a
  // small remainder that leaves most of the GPU idle
  const long long max_entries = 48ll << 20;
  int zchunk = (int)(max_entries / (plane * GF_NA));
  if (zchunk < 1) zchunk = 1;
  if (zchunk > z1 - z0) zchunk = z1 - z0;
  const int nchunks = (z1 - z0 + zchunk - 1) / zchunk;
  zchunk = (z1 - z0 + nchunks - 1) / nchunks;
  // float maps: phase A keeps the partial MCC of the voxels with eigen-tasks in float64 (zchunk planes), so the finished
  // MCC is rounded to float once
  constexpr bool f64 = std::is_same<OutT, double>::value;
  const size_t ntasks = (size_t)zchunk * plane * GF_NA, nmcc = f64 ? 0 : (size_t)zchunk * plane;
  std::unique_lock<std::mutex> lk;       // held until the last chunk's finish kernel is enqueued
  StreamScratch* S = stream_scratch(st, lk);
  if (!S || !S->grow(S->count, sizeof(unsigned)) || !S->grow(S->tasks, ntasks * sizeof(GlcmTask)) ||
      !S->grow(S->results, ntasks * sizeof(double)) || !S->grow(S->mcc, nmcc * sizeof(double)))
    return fail(RB_ERR_NOMEM, "could not allocate the GLCM eigen-task queue");
  GlcmTask* q = S->tasks.as<GlcmTask>();
  double *res = S->results.as<double>(), *mcc = S->mcc.as<double>();
  unsigned* count = S->count.as<unsigned>();
  // phase A: one CTA per SM (register-bound).  512 threads at 128 registers (a hundred spilled words per thread, L1-
  // resident) put 16 warps on an SM instead of the 8 of a 256-thread / 236-register build, which hides more of the
  // latency of this issue-bound kernel.
  constexpr int NT = 512;
  const int smem = glcm_phaseA_smem_bytes(NT);
  RB_CUDA(set_max_dynamic_smem(glcm_fast_kernel<1, NT, OutT>, smem));
  // register Lanczos: 90 KB of per-thread shared vectors per CTA -> two CTAs per SM
  RB_CUDA(set_max_dynamic_smem(glcm_fast_solve_kernel<2>, GF_LZ_SMEM_BYTES));
  for (int za = z0; za < z1; za += zchunk) {
    const int zb = za + zchunk < z1 ? za + zchunk : z1;
    RB_CUDA(cudaMemsetAsync(count, 0, sizeof(unsigned), st));
    int grid = 0;
    RB_CUDA(resident_grid(glcm_fast_kernel<1, NT, OutT>, NT, smem, (long long)(zb - za) * plane, grid));
    glcm_fast_kernel<1, NT, OutT><<<grid, NT, smem, st>>>(l8, centers, P, T, out, fstride, za, zb, out_z0, q, count, mcc);
    RB_LAUNCH_CHECK();
    // One launch per size group keeps ONE solver body in the instruction cache (the three Lanczos templates together are
    // 18.5 k SASS instructions, 296 KB, and on a smooth volume the blocks of an SM otherwise sit in different groups); the
    // dense n <= 8 solves stay a single launch, where the repeated tile sorts would cost more than they save.
    glcm_fast_solve_kernel<0><<<sms * 8, 128, 0, st>>>(l8, P, T, q, count, res, 0);
    for (int g = 10; g <= 12; g += 2) glcm_fast_solve_kernel<1><<<sms * 8, 128, 0, st>>>(l8, P, T, q, count, res, g);
    for (int g = 18; g >= 14; g -= 2)
      glcm_fast_solve_kernel<2><<<sms * 2, 128, GF_LZ_SMEM_BYTES, st>>>(l8, P, T, q, count, res, g);
    RB_LAUNCH_CHECK();
    glcm_fast_finish_kernel<OutT><<<sms * 8, 256, 0, st>>>(P, q, count, res, out + (long long)G_MCC * fstride,
                                                           out_z0, mcc, za);
    RB_LAUNCH_CHECK();
  }
  return RB_OK;
}

// ---------------------------------------------------------------------------------- GLRLM
template <typename OutT>
__global__ void __launch_bounds__(128)
glrlm_fast_kernel(const uint8_t* __restrict__ lev, const uint8_t* __restrict__ centers,
                  const __grid_constant__ VoxParams P, const GlrlmFastTables* __restrict__ Tg,
                  OutT* __restrict__ out, long long fstride, int z0, int z1, int out_z0) {
  __shared__ GlrlmFastTables T;
  copy_tables_to_shared(T, Tg);
  __syncthreads();
  const long long plane = (long long)P.Y * P.X;
  const long long total = (long long)(z1 - z0) * plane;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const ChunkVoxel v = chunk_voxel(P, plane, z0, out_z0, t);
    if (!chunk_center(lev, centers, plane, v)) {
#pragma unroll
      for (int k = 0; k < GLRLM_NF; k++) store_map(out + k * fstride + v.oi, P.init_value);
      continue;
    }
    int wl[27];
    load_window27(lev, P, v.z, v.y, v.x, v.vi, true, wl, 1);
    double f[GLRLM_NF];
    glrlm_fast_voxel(wl, T, f);
#pragma unroll
    for (int k = 0; k < GLRLM_NF; k++) store_map(out + k * fstride + v.oi, f[k]);
  }
}

template <typename OutT>
static int glrlm_fast_run(const uint8_t* l8, const uint8_t* centers, const VoxParams& P, OutT* out, long long fstride,
                          int z0, int z1, int out_z0, cudaStream_t st) {
  const GlrlmFastTables* T = device_table<GlrlmFastTables>(glrlm_fast_build_tables);
  if (!T) return fail(RB_ERR_CUDA, "could not build the GLRLM table block on the device");
  const long long total = (long long)(z1 - z0) * P.Y * P.X;
  if (total <= 0) return RB_OK;
  glrlm_fast_kernel<<<grid_for(total, 128, 32), 128, 0, st>>>(l8, centers, P, T, out, fstride, z0, z1, out_z0);
  RB_LAUNCH_CHECK();
  return RB_OK;
}

// ------------------------------------------------------------------ GLSZM / GLDM / NGTDM fast paths
// One tile kernel over the full/deferred tiles of full_window_tiles (voxel_tiles.cuh): a centre whose 27 window levels
// are all non-zero runs the class's full-window body in its tile, the other centres are drained through its general
// body.  Per class: the feature count, the block size NT and blocks per SM MINB (registers <= 65536 / (NT * MINB): 16
// warps per SM), the per-thread shared scratch of the level classes, laid out [entry][thread], and the two bodies.
template <int CLS> struct TileClass;
template <> struct TileClass<C_GLSZM> {
  static constexpr int NF = GLSZM_NF, NT = 128, MINB = 4;
  struct Scratch { unsigned long long mg[13 * NT]; };                 // mask | level << 32 of each repeated level
  template <bool FULL>
  static __device__ __forceinline__ void body(const int* wl, const SmallFastTables& T, int, Scratch& s, int tid, double* f) {
    glszm_fast_body<FULL>(wl, T, f, s.mg + tid, NT);
  }
};
template <> struct TileClass<C_GLDM> {
  static constexpr int NF = GLDM_NF, NT = 256, MINB = 2;
  struct Scratch {};
  template <bool FULL>
  static __device__ __forceinline__ void body(const int* wl, const SmallFastTables& T, int alpha, Scratch&, int, double* f) {
    gldm_fast_body<FULL>(wl, alpha, T, f);
  }
};
template <> struct TileClass<C_NGTDM> {
  static constexpr int NF = NGTDM_NF, NT = 128, MINB = 4;
  struct Scratch { double ns[27 * NT]; int pk[27 * NT]; };            // per-class diff sums, then the compacted classes
  template <bool FULL>
  static __device__ __forceinline__ void body(const int* wl, const SmallFastTables& T, int, Scratch& s, int tid, double* f) {
    ngtdm_fast_body<FULL>(wl, T, f, s.pk + tid, s.ns + tid, NT);
  }
};

template <int CLS, int NT, int MINB, typename OutT>
__global__ void __launch_bounds__(NT, MINB)
tiles_fast_kernel(const uint8_t* __restrict__ lev, const uint8_t* __restrict__ centers, const __grid_constant__ VoxParams P,
                  const SmallFastTables* __restrict__ Tg, OutT* __restrict__ out, long long fstride,
                  int z0, int z1, int out_z0) {
  using K = TileClass<CLS>;
  static_assert(NT == K::NT && MINB == K::MINB, "the scratch is laid out for the class's block size");
  __shared__ SmallFastTables T;
  __shared__ typename K::Scratch scr;
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
      const bool full = load_window27(lev, P, v.z, v.y, v.x, v.vi, is_center, wl, 1);
      if (full) {
        double f[K::NF];
        K::template body<true>(wl, T, P.alpha, scr, tid, f);
#pragma unroll
        for (int k = 0; k < K::NF; k++) store_map(out + k * fstride + v.oi, f[k]);
      } else if (is_center) {
        defer_it();
      } else {
#pragma unroll
        for (int k = 0; k < K::NF; k++) store_map(out + k * fstride + v.oi, P.init_value);
      }
    },
    [&](auto entry, bool live) {
      if (!live) return;
      const ChunkVoxel v = chunk_voxel(P, plane, z0, out_z0, entry());
      int wl[27];
      load_window27(lev, P, v.z, v.y, v.x, v.vi, true, wl, 1);
      double f[K::NF];
      K::template body<false>(wl, T, P.alpha, scr, tid, f);
#pragma unroll
      for (int k = 0; k < K::NF; k++) store_map(out + k * fstride + v.oi, f[k]);
    });
}

template <int CLS, typename OutT>
static int tiles_fast_run(const uint8_t* l8, const uint8_t* centers, const VoxParams& P, OutT* out, long long fstride,
                          int z0, int z1, int out_z0, cudaStream_t st) {
  using K = TileClass<CLS>;
  const SmallFastTables* T = device_table<SmallFastTables>(small_fast_build_tables);
  if (!T) return fail(RB_ERR_CUDA, "could not build the table block on the device");
  const long long total = (long long)(z1 - z0) * P.Y * P.X;
  if (total <= 0) return RB_OK;
  int grid = 0;
  RB_CUDA(resident_grid(tiles_fast_kernel<CLS, K::NT, K::MINB, OutT>, K::NT, 0, total, grid));
  tiles_fast_kernel<CLS, K::NT, K::MINB, OutT><<<grid, K::NT, 0, st>>>(l8, centers, P, T, out, fstride, z0, z1, out_z0);
  RB_LAUNCH_CHECK();
  return RB_OK;
}

// ------------------------------------------------------------------------------------ the entry
// the fast kernels of class A.cls, for settings voxel_fast_path (host_common.hpp) accepts
int voxel_fast_launch(const VoxLaunch& A) {
  return with_map_type(A.out_f32, [&](auto ot) -> int {
    using OutT = decltype(ot);
    const uint8_t* l8 = (const uint8_t*)A.lev;
    OutT* out = (OutT*)A.out;
    switch (A.cls) {
      case C_GLCM: return glcm_fast_run(l8, A.centers, A.P, out, A.fstride, A.z0, A.z1, A.out_z0, A.st);
      case C_GLRLM: return glrlm_fast_run(l8, A.centers, A.P, out, A.fstride, A.z0, A.z1, A.out_z0, A.st);
      case C_GLSZM: return tiles_fast_run<C_GLSZM>(l8, A.centers, A.P, out, A.fstride, A.z0, A.z1, A.out_z0, A.st);
      case C_GLDM: return tiles_fast_run<C_GLDM>(l8, A.centers, A.P, out, A.fstride, A.z0, A.z1, A.out_z0, A.st);
      default: return tiles_fast_run<C_NGTDM>(l8, A.centers, A.P, out, A.fstride, A.z0, A.z1, A.out_z0, A.st);
    }
  });
}

}  // namespace rb
