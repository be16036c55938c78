// The kernels of the fused GLCM path as a header: the eigen-task queue entry, phase A (per-voxel features +
// task queue), the three solve kernels (phase B) and the finish kernel (phase C).
// Split from voxel_fast.cu so that tests/host_emul/solve_kernel_emul.cpp can compile the SAME kernel text for
// the CPU (one std::thread per CUDA thread, barriers as barriers) and check its tile sort / grouping / barrier
// structure -- and race-check it with ThreadSanitizer -- without a GPU.
#pragma once
#include "glcm_fast.cuh"
#include "voxel_tiles.cuh"

#ifndef RB_DYN_SHARED          // dynamic shared memory of the launching kernel
#define RB_DYN_SHARED(type, name) extern __shared__ type name[]
#endif

namespace rb {

// Two kernels per chunk of planes:
//   A  one thread per centre voxel: window -> equality masks -> all 13 angles, every feature except
//      the MCC eigen-solves; a voxel that needs k solves reserves k CONSECUTIVE 16-byte queue entries
//      (voxel, angle slot, n_ok).
//   B  one thread per queue entry (= one eigen-task): reloads the voxel's 27 levels and runs the dense register
//      solve (<= 12 levels) or the register-resident Lanczos recurrence (13..18 levels); result to res[k].
//   C  one thread per voxel-with-tasks adds its results in slot order to the voxel's MCC (single
//      writer, fixed order: deterministic).  Eigen-solves are needed by a few % of the
//      (voxel, angle) pairs on noisy data and by most on smooth data; left inline they idle most
//      lanes of a warp behind one long solve and force 255 registers on every thread.
struct GlcmTask {
  long long vi;        // linear index of the voxel in the level volume
  uint8_t slot;        // angle slot to solve
  uint8_t n_ok;        // number of non-empty angles of the voxel (the nanmean denominator)
  uint8_t count;       // > 0 on the first task of a voxel: how many consecutive entries belong to it
  uint8_t cls;         // size class of the task (glcm_task_class), groups similar tasks in a warp
  float unused;
};

// Phase B.  KIND 0: tasks with n <= 8 levels, KIND 1: 9..12 (dense register solves, see glcm_small_solve),
// KIND 2: larger level graphs (register Lanczos, glcm_lanczos.cuh; dynamic shared memory = LZ_NARR * 18 doubles per
// thread).  Each is its own kernel because the three want very different register budgets.
constexpr int GF_LZ_SMEM_BYTES = LZ_NARR * 18 * 128 * (int)sizeof(double);
constexpr int glcm_phaseA_smem_bytes(int nt) { return 27 * nt * (int)(sizeof(uint32_t) + sizeof(uint8_t)); }
template <int KIND> struct SolveKind;
template <> struct SolveKind<0> { static constexpr int lo = 0, hi = 6, minb = 4; };
template <> struct SolveKind<1> { static constexpr int lo = 7, hi = GF_DENSE_MAX_CLS, minb = 2; };
template <> struct SolveKind<2> { static constexpr int lo = GF_DENSE_MAX_CLS + 1, hi = GF_NCLS - 1, minb = 2; };

// the 27 window levels of the voxel with linear index vi (zeros if !live)
__device__ __forceinline__ void glcm_task_window(const uint8_t* __restrict__ lev, const VoxParams& P, long long vi, bool live,
                                                 uint8_t* w) {
  const int z = (int)(vi / P.sz), rem = (int)(vi % P.sz), y = rem / (int)P.sy, x = rem % (int)P.sy;
  load_window27(lev, P, z, y, x, vi, live, w, 1);
}

// sorted positions [begin, end) of the tile: tasks whose level graph has at most N nodes
template <int N>
__device__ __forceinline__ void solve_group(const uint8_t* __restrict__ lev, const VoxParams& P, const GlcmSolveTables& T,
                                            const GlcmTask* __restrict__ queue, double* __restrict__ res,
                                            const uint16_t* order, unsigned base, int begin, int end) {
  for (int b0 = begin; b0 < end; b0 += 128) {              // block-uniform bounds
    const int i = b0 + (int)threadIdx.x;
    const bool live = i < end;
    const unsigned k = base + order[live ? i : begin];
    const GlcmTask e = queue[k];
    uint8_t w[27];
    glcm_task_window(lev, P, e.vi, live, w);
    uint32_t W7[7];
    glcm_pack_window(w, 1, W7);
    bool ok;
    const double r = glcm_small_solve<N, true>(w, 1, W7, T, e.slot, &ok, live);
    if (live) res[k] = ok ? r : NAN;
  }
}

// sorted positions [begin, end) of the tile: large tasks whose level graph has at most N nodes (N = 14 / 16 / 18)
template <int N>
__device__ __forceinline__ void lanczos_group(const uint8_t* __restrict__ lev, const VoxParams& P, const GlcmSolveTables& T,
                                              const GlcmTask* __restrict__ queue, double* __restrict__ res,
                                              const uint16_t* order, unsigned base, int begin, int end, double* scratch) {
  for (int b0 = begin; b0 < end; b0 += 128) {
    const int i = b0 + (int)threadIdx.x;
    if (b0 + (int)(threadIdx.x & ~31u) >= end) break;   // a warp with no task left (the solver holds no barrier)
    const bool live = i < end;
    const unsigned k = base + order[live ? i : begin];
    const GlcmTask e = queue[k];
    uint8_t w[27];
    glcm_task_window(lev, P, e.vi, live, w);
    int n = 0;
    double r = e.slot <= 2 ? glcm_lanczos_task<N>(w, 1, T, e.slot, scratch + threadIdx.x, 128, &n, live) : 1.0;
    if (N == 18 && n == 19) r = 1.0;            // a tree (see glcm_lanczos_solve); phase A does not queue these
    if (live) res[k] = r;
  }
}

template <int KIND>
__global__ void __launch_bounds__(128, SolveKind<KIND>::minb)
glcm_fast_solve_kernel(const uint8_t* __restrict__ lev, const __grid_constant__ VoxParams P,
                       const GlcmFastTables* __restrict__ Tg, const GlcmTask* __restrict__ queue,
                       const unsigned* __restrict__ qcount, double* __restrict__ res, int only) {
  // only = 0: every size group of this kind; else just the group of that template size (one launch per group keeps ONE
  // solver body in the instruction cache at a time: on smooth volumes the blocks of an SM sit in different groups)
  __shared__ GlcmSolveTables T;
  if (threadIdx.x == 0) glcm_solve_tables_from(*Tg, T);
  __syncthreads();
  const unsigned n = *qcount;
  // Tiles of up to 4096 consecutive tasks are counting-sorted by size class in shared memory, so the lanes of a warp run
  // solves of the same size (otherwise a third of the lanes stay active).  The sort is STABLE and atomic-free (per-thread
  // counts, one serial scan per class), so a task's position is the same in every run.  The Lanczos kind cuts the queue
  // into a whole number of tiles per block, all of one size (+-1), so no launch ends on a partial wave of tiles; the dense
  // kinds, whose block-uniform rounds cost the same however few tasks they hold, keep full tiles.  A task's result does
  // not depend on its tile.
  constexpr int TILE = 4096;
  constexpr int LO = SolveKind<KIND>::lo, KC = SolveKind<KIND>::hi - SolveKind<KIND>::lo + 1;
  __shared__ uint16_t order[TILE];
  __shared__ int bucket[GF_NCLS];                 // end position of each class of this kind in `order`
  __shared__ uint16_t cnt[KC][128];               // [class][thread]: count, then exclusive prefix over the threads
  const unsigned long long per_wave = (unsigned long long)gridDim.x * TILE;
  const unsigned ntiles = KIND == 2 ? gridDim.x * (unsigned)((n + per_wave - 1) / per_wave) : (n + TILE - 1) / TILE;
  for (unsigned tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const unsigned base = KIND == 2 ? (unsigned)((unsigned long long)n * tile / ntiles) : tile * TILE;
    const unsigned tend = KIND == 2 ? (unsigned)((unsigned long long)n * (tile + 1) / ntiles)   // tend - base <= TILE
                                    : (n - base < (unsigned)TILE ? n : base + TILE);
#pragma unroll
    for (int c = 0; c < KC; c++) cnt[c][threadIdx.x] = 0;
    if (threadIdx.x < GF_NCLS) bucket[threadIdx.x] = 0;
    uint8_t mycls[TILE / 128];
#pragma unroll
    for (int j = 0; j < TILE / 128; j++) {
      const unsigned k = base + j * 128 + threadIdx.x;
      mycls[j] = k < tend ? queue[k].cls : GF_NCLS;
      const int c = (int)mycls[j] - LO;
      if (c >= 0 && c < KC) cnt[c][threadIdx.x]++;
    }
    __syncthreads();
    if ((int)threadIdx.x < KC) {                   // one thread per class: exclusive scan over the 128 per-thread counts
      int run = 0;
      for (int t = 0; t < 128; t++) { const int v = cnt[threadIdx.x][t]; cnt[threadIdx.x][t] = (uint16_t)run; run += v; }
      bucket[LO + threadIdx.x] = run;              // class total (turned into the class end below)
    }
    __syncthreads();
    int cstart[KC];                                // start of each class = totals of the smaller classes
    {
      int run = 0;
#pragma unroll
      for (int c = 0; c < KC; c++) { cstart[c] = run; run += bucket[LO + c]; }
    }
    __syncthreads();
    if ((int)threadIdx.x < KC) bucket[LO + threadIdx.x] += cstart[threadIdx.x];
#pragma unroll
    for (int j = 0; j < TILE / 128; j++) {
      const int c = (int)mycls[j] - LO;
      if (c >= 0 && c < KC) {
        int cs = 0;
#pragma unroll
        for (int q = 0; q < KC; q++) if (q == c) cs = cstart[q];
        order[cs + cnt[c][threadIdx.x]++] = (uint16_t)(j * 128 + threadIdx.x);
      }
    }
    __syncthreads();
    if (KIND == 2) {
      RB_DYN_SHARED(double, lz_scratch);                 // [LZ_NARR * 18][128]
      // size groups from the top: a task's size class fixes the template that solves it
      const int e14 = bucket[12], e16 = bucket[14], e18 = bucket[15];
      if (!only || only == 18) lanczos_group<18>(lev, P, T, queue, res, order, base, e16, e18, lz_scratch);
      if (!only || only == 16) lanczos_group<16>(lev, P, T, queue, res, order, base, e14, e16, lz_scratch);
      if (!only || only == 14) lanczos_group<14>(lev, P, T, queue, res, order, base, 0, e14, lz_scratch);
    } else {
      // dense solves: one template size at a time, block-uniform (idle threads run on an empty window), so the
      // barriers inside glcm_small_solve keep the warps on the same code (free-running warps stall on instruction
      // fetch -- these bodies are 2-10 k straight-line instructions)
      if (KIND == 0) {
        if (!only || only == 4) solve_group<4>(lev, P, T, queue, res, order, base, 0, bucket[2]);
        if (!only || only == 6) solve_group<6>(lev, P, T, queue, res, order, base, bucket[2], bucket[4]);
        if (!only || only == 8) solve_group<8>(lev, P, T, queue, res, order, base, bucket[4], bucket[6]);
      } else {
        if (!only || only == 10) solve_group<10>(lev, P, T, queue, res, order, base, 0, bucket[8]);
        if (!only || only == 12) solve_group<12>(lev, P, T, queue, res, order, base, bucket[8], bucket[GF_DENSE_MAX_CLS]);
      }
    }
    __syncthreads();
  }
}

// ---- phase A (one thread per centre voxel) and phase C (finish) ---------------------------------
// phase A of one centre voxel; store: write its 24 maps and queue its eigen-tasks (the general body holds barriers, so
// every thread of the block runs it, idle ones with store = false).  Float maps: the partial MCC of a voxel with tasks
// also goes to mcc_part[t] (t = chunk index) in double, so that phase C rounds the finished MCC once.
template <bool FULL, int NT, typename OutT>
__device__ __forceinline__ void glcm_phaseA_voxel(const uint8_t* w, uint32_t* eq, const GlcmFastTables& T, const VoxParams& P,
                                                  const ChunkVoxel& v, bool store, OutT* __restrict__ out, long long fstride,
                                                  GlcmTask* __restrict__ queue, unsigned* __restrict__ qcount,
                                                  double* __restrict__ mcc_part, long long t) {
  double f[GLCM_NF];
  int n_ok = 0;
  unsigned long long tcls = 0;
  const uint32_t tasks = glcm_fast_voxel_phaseA<FULL>(w, NT, eq, NT, T, P, f, &n_ok, &tcls);
  if (!store) return;
#pragma unroll
  for (int k = 0; k < GLCM_NF; k++) store_map(out + k * fstride + v.oi, f[k]);
  if constexpr (!std::is_same<OutT, double>::value) {
    if (tasks) mcc_part[t] = f[G_MCC];
  }
  if (tasks) {
    const int k = __popc(tasks);
    unsigned q = atomicAdd(qcount, (unsigned)k);
    bool first = true;
    for (uint32_t m = tasks; m; m &= m - 1, q++) {
      GlcmTask e;
      e.vi = v.vi; e.slot = (uint8_t)(__ffs((int)m) - 1); e.n_ok = (uint8_t)n_ok; e.count = first ? (uint8_t)k : 0;
      e.cls = (uint8_t)(tcls >> (GF_CLS_BITS * e.slot) & (GF_NCLS - 1)); e.unused = 0.f;
      queue[q] = e;
      first = false;
    }
  }
}

// Phase A over the full/deferred tiles of full_window_tiles (voxel_tiles.cuh).  The window bytes live in shared
// memory, [27][NT].  (List entries are chunk indices: a chunk of 2^32 voxels would need a 1.3 TB eigen-task queue,
// which glcm_fast_run fails to allocate first.)
// OutT: the map type (store_map).  mcc_part: the chunk's float64 partial-MCC plane, float maps only.
template <int MINB, int NT, typename OutT>
__global__ void __launch_bounds__(NT, MINB)
glcm_fast_kernel(const uint8_t* __restrict__ lev, const uint8_t* __restrict__ centers,
                 const __grid_constant__ VoxParams P, const GlcmFastTables* __restrict__ Tg,
                 OutT* __restrict__ out, long long fstride, int z0, int z1, int out_z0,
                 GlcmTask* __restrict__ queue, unsigned* __restrict__ qcount, double* __restrict__ mcc_part = nullptr) {
  __shared__ GlcmFastTables T;
  __shared__ unsigned defer[2 * NT];                                // chunk indices of the voxels left to the general body
  __shared__ unsigned ndefer;
  RB_DYN_SHARED(uint32_t, eqbuf);                                   // [27][NT] equality masks, then [27][NT] window bytes
  uint8_t* const wbuf = reinterpret_cast<uint8_t*>(eqbuf + 27 * NT);
  copy_tables_to_shared<NT>(T, Tg);
  if (threadIdx.x == 0) ndefer = 0;
  __syncthreads();
  uint8_t* const w = &wbuf[threadIdx.x];
  uint32_t* const eq = &eqbuf[threadIdx.x];
  full_window_tiles<NT>((long long)(z1 - z0) * P.Y * P.X, defer, ndefer,
    [&](long long t, bool live, auto defer_it) {
      const long long plane = (long long)P.Y * P.X;
      const ChunkVoxel v = chunk_voxel(P, plane, z0, out_z0, t, live);
      const bool center = live && chunk_center(lev, centers, plane, v);
      if (load_window27(lev, P, v.z, v.y, v.x, v.vi, center, w, NT)) {
        glcm_phaseA_voxel<true, NT>(w, eq, T, P, v, true, out, fstride, queue, qcount, mcc_part, t);
      } else if (center) {
        defer_it();
      } else if (live) {
#pragma unroll
        for (int k = 0; k < GLCM_NF; k++) store_map(out + k * fstride + v.oi, P.init_value);
      }
    },
    [&](auto entry, bool live) {                                    // idle threads run on an all-zero window
      const long long plane = (long long)P.Y * P.X;
      const long long t = live ? entry() : 0;
      const ChunkVoxel v = chunk_voxel(P, plane, z0, out_z0, t, live);
      load_window27(lev, P, v.z, v.y, v.x, v.vi, live && chunk_center(lev, centers, plane, v), w, NT);
      glcm_phaseA_voxel<false, NT>(w, eq, T, P, v, live, out, fstride, queue, qcount, mcc_part, t);
    });
}


// Float maps: the partial MCC comes from phase A's float64 plane mcc_part (chunk of planes from za), and the finished
// double sum is rounded once as it is stored.
template <typename OutT>
__global__ void __launch_bounds__(256)
glcm_fast_finish_kernel(const __grid_constant__ VoxParams P, const GlcmTask* __restrict__ queue,
                        const unsigned* __restrict__ qcount, const double* __restrict__ res,
                        OutT* __restrict__ mcc_map /* out + G_MCC*fstride */, int out_z0,
                        const double* __restrict__ mcc_part = nullptr, int za = 0) {
  const unsigned n = *qcount;
  const long long plane = (long long)P.Y * P.X;
  for (unsigned k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const GlcmTask e = queue[k];
    if (!e.count) continue;
    double add = 0;
    for (int j = 0; j < e.count; j++) add += res[k + j];
    const long long oi = e.vi - (long long)out_z0 * plane;   // contiguous volume: vi = z*plane + rem
    if constexpr (std::is_same<OutT, double>::value) mcc_map[oi] += add / e.n_ok;
    else {
      const double mcc = mcc_part[e.vi - (long long)za * plane] + add / e.n_ok;
      store_map(mcc_map + oi, mcc);
    }
  }
}

}  // namespace rb
