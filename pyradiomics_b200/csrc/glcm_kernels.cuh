// The kernels of the fused GLCM path as a header: the eigen-task queue entry, phase A (per-voxel features +
// task queue), the three solve kernels (phase B) and the finish kernel (phase C).
// Split from voxel_fast.cu so that tests/host_emul/solve_kernel_emul.cpp can compile the SAME kernel text for
// the CPU (one std::thread per CUDA thread, barriers as barriers) and check its tile sort / grouping / barrier
// structure -- and race-check it with ThreadSanitizer -- without a GPU.
#pragma once
#include "glcm_fast.cuh"

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
#ifndef GF_DENSE_SYNC
#define GF_DENSE_SYNC 1
#endif
#ifndef GF_SOLVE_MINB_S
#define GF_SOLVE_MINB_S 4
#endif
#ifndef GF_SOLVE_MINB_L
#define GF_SOLVE_MINB_L 2
#endif
#ifndef GF_LZ_TOPUP
#define GF_LZ_TOPUP 0              // 1: a size group's last batch is topped up with tasks of the next smaller group (needs
                                   // LZ_EIG_EXACT_STATIC = 0 for reproducible bits)
#endif
static_assert(!(GF_LZ_TOPUP && LZ_EIG_EXACT_STATIC), "topped-up batches need the task-sized eigenvalue search (LZ_EIG_EXACT_STATIC=0): "
                                                      "otherwise a task's bits depend on the template that happens to solve it");
#ifndef GF_SOLVE_TILE
#define GF_SOLVE_TILE 4096
#endif
constexpr int GF_LZ_SMEM_BYTES = LZ_NARR * 18 * 128 * (int)sizeof(double);
constexpr int glcm_phaseA_smem_bytes(int nt) { return 27 * nt * (int)(sizeof(uint32_t) + sizeof(uint8_t)); }
template <int KIND> struct SolveKind;
template <> struct SolveKind<0> { static constexpr int lo = 0, hi = 6, minb = GF_SOLVE_MINB_S; };
template <> struct SolveKind<1> { static constexpr int lo = 7, hi = GF_DENSE_MAX_CLS, minb = 2; };
template <> struct SolveKind<2> { static constexpr int lo = GF_DENSE_MAX_CLS + 1, hi = GF_NCLS - 1, minb = GF_SOLVE_MINB_L; };

// the 27 window levels of the voxel with linear index vi (zeros if !live)
__device__ __forceinline__ void glcm_task_window(const uint8_t* __restrict__ lev, const VoxParams& P, long long vi, bool live,
                                                 uint8_t* w) {
  const int z = (int)(vi / P.sz), rem = (int)(vi % P.sz), y = rem / (int)P.sy, x = rem % (int)P.sy;
  int p = 0;
#pragma unroll
  for (int dz = -1; dz <= 1; dz++)
#pragma unroll
    for (int dy = -1; dy <= 1; dy++)
#pragma unroll
      for (int dx = -1; dx <= 1; dx++, p++) {
        const int zz = z + dz, yy = y + dy, xx = x + dx;
        const bool in = live && zz >= 0 && zz < P.Z && yy >= 0 && yy < P.Y && xx >= 0 && xx < P.X;
        w[p] = in ? lev[vi + (long long)dz * P.sz + (long long)dy * P.sy + dx] : (uint8_t)0;
      }
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
    const double r = glcm_small_solve<N, GF_DENSE_SYNC != 0>(w, 1, W7, T, e.slot, &ok, live);
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
  // Tiles of GF_SOLVE_TILE (4096) consecutive tasks are counting-sorted by size class in shared memory, so the
  // lanes of a warp run solves of the same size (otherwise a third of the lanes stay active).  The sort is STABLE and
  // atomic-free (per-thread counts, one serial scan per class), so the position of a task -- and with it the batch and,
  // for topped-up Lanczos batches, the size template that solves it -- is the same in every run: bit-reproducible maps.
  constexpr int TILE = GF_SOLVE_TILE;
  constexpr int LO = SolveKind<KIND>::lo, KC = SolveKind<KIND>::hi - SolveKind<KIND>::lo + 1;
  __shared__ uint16_t order[TILE];
  __shared__ int bucket[GF_NCLS];                 // end position of each class of this kind in `order`
  __shared__ uint16_t cnt[KC][128];               // [class][thread]: count, then exclusive prefix over the threads
  const unsigned ntiles = (n + TILE - 1) / TILE;
  for (unsigned tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const unsigned base = tile * TILE;
#pragma unroll
    for (int c = 0; c < KC; c++) cnt[c][threadIdx.x] = 0;
    if (threadIdx.x < GF_NCLS) bucket[threadIdx.x] = 0;
    uint8_t mycls[TILE / 128];
#pragma unroll
    for (int j = 0; j < TILE / 128; j++) {
      const unsigned k = base + j * 128 + threadIdx.x;
      mycls[j] = k < n ? queue[k].cls : GF_NCLS;
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
      // size groups from the top; a group's last batch is topped up with tasks of the next smaller group (a larger N
      // solves them as well: padded nodes), so a tile has ONE partially filled batch instead of three
      const int e14 = bucket[12], e16 = bucket[14], e18 = bucket[15];
      int s18 = GF_LZ_TOPUP ? e18 - (e18 - e16 + 127) / 128 * 128 : e16;
      if (s18 < 0) s18 = 0;
      const int e16b = s18 < e16 ? s18 : e16;
      int s16 = !GF_LZ_TOPUP ? e14 : e16b > e14 ? e16b - (e16b - e14 + 127) / 128 * 128 : e16b;
      if (s16 < 0) s16 = 0;
      const int e14b = s16 < e14 ? s16 : e14;
      if (!only || only == 18) lanczos_group<18>(lev, P, T, queue, res, order, base, s18, e18, lz_scratch);
      if (!only || only == 16) lanczos_group<16>(lev, P, T, queue, res, order, base, s16, e16b, lz_scratch);
      if (!only || only == 14) lanczos_group<14>(lev, P, T, queue, res, order, base, 0, e14b, lz_scratch);
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
struct PhaseAVoxel { long long vi, oi; bool center, full; };

// voxel t of the chunk: its 27 window levels to w (stride NT; zeros outside the volume, all zeros if it is not a
// centre) and whether the window is full (a centre whose 27 levels are all non-zero, see glcm_window_full)
template <int NT>
__device__ __forceinline__ PhaseAVoxel glcm_phaseA_load(const uint8_t* __restrict__ lev, const uint8_t* __restrict__ centers,
                                                        const VoxParams& P, int z0, int out_z0, long long t, bool live,
                                                        uint8_t* w) {
  const long long plane = (long long)P.Y * P.X;
  const int z = z0 + (int)((live ? t : 0) / plane);
  const int rem = (int)((live ? t : 0) % plane);
  const int y = rem / P.X, x = rem % P.X;
  PhaseAVoxel v;
  v.vi = (long long)z * P.sz + (long long)y * P.sy + x;
  v.oi = (long long)(z - out_z0) * plane + rem;
  v.center = live && (centers ? centers[(long long)z * plane + rem] != 0 : lev[v.vi] != 0);
  bool full = v.center;
#pragma unroll
  for (int dz = -1; dz <= 1; dz++)
#pragma unroll
    for (int dy = -1; dy <= 1; dy++)
#pragma unroll
      for (int dx = -1; dx <= 1; dx++) {
        const int zz = z + dz, yy = y + dy, xx = x + dx;
        const bool in = v.center && zz >= 0 && zz < P.Z && yy >= 0 && yy < P.Y && xx >= 0 && xx < P.X;
        const uint8_t l = in ? lev[v.vi + (long long)dz * P.sz + (long long)dy * P.sy + dx] : (uint8_t)0;
        full &= l != 0;
        w[((dz + 1) * 9 + (dy + 1) * 3 + (dx + 1)) * NT] = l;
      }
  v.full = full;
  return v;
}

// phase A of one centre voxel; store: write its 24 maps and queue its eigen-tasks (the general body holds barriers, so
// every thread of the block runs it, idle ones with store = false)
template <bool FULL, int NT>
__device__ __forceinline__ void glcm_phaseA_voxel(const uint8_t* w, uint32_t* eq, const GlcmFastTables& T, const VoxParams& P,
                                                  const PhaseAVoxel& v, bool store, double* __restrict__ out, long long fstride,
                                                  GlcmTask* __restrict__ queue, unsigned* __restrict__ qcount) {
  double f[GLCM_NF];
  int n_ok = 0;
  unsigned long long tcls = 0;
  const uint32_t tasks = glcm_fast_voxel_phaseA<FULL>(w, NT, eq, NT, T, P, f, &n_ok, &tcls);
  if (!store) return;
#pragma unroll
  for (int k = 0; k < GLCM_NF; k++) out[k * fstride + v.oi] = f[k];
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

// Block-uniform tiles of NT voxels: a centre with a full window runs the full-window body (no validity logic, constant
// denominators, no barriers), a voxel that is not a centre stores init_value, and a centre whose window is not full (the
// volume's faces, the ROI's border and holes) goes to the block's list.  The block runs the general body over that
// list, NT at a time, whenever NT are waiting and once at the end.  (List entries are chunk indices: a chunk of 2^32
// voxels would need a 1.3 TB eigen-task queue, which glcm_fast_launch fails to allocate first.)
template <int MINB, int NT>
__global__ void __launch_bounds__(NT, MINB)
glcm_fast_kernel(const uint8_t* __restrict__ lev, const uint8_t* __restrict__ centers,
                 const __grid_constant__ VoxParams P, const GlcmFastTables* __restrict__ Tg,
                 double* __restrict__ out, long long fstride, int z0, int z1, int out_z0,
                 GlcmTask* __restrict__ queue, unsigned* __restrict__ qcount) {
  __shared__ GlcmFastTables T;
  __shared__ unsigned defer[2 * NT];                                // chunk indices of the voxels left to the general body
  __shared__ unsigned ndefer;
  RB_DYN_SHARED(uint32_t, eqbuf);                                   // [27][NT] equality masks, then [27][NT] window bytes
  uint8_t* const wbuf = reinterpret_cast<uint8_t*>(eqbuf + 27 * NT);
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(Tg);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&T);
    for (int i = threadIdx.x; i < (int)(sizeof(GlcmFastTables) / 4); i += NT) dst[i] = src[i];
  }
  const int tid = threadIdx.x;
  if (tid == 0) ndefer = 0;
  __syncthreads();
  const long long total = (long long)(z1 - z0) * P.Y * P.X;
  const long long ntiles = (total + NT - 1) / NT;
  uint8_t* const w = &wbuf[tid];
  uint32_t* const eq = &eqbuf[tid];
  // one pass per tile and a last pass with no tile (one call site per body: each is thousands of instructions)
  for (long long tile = blockIdx.x;; tile += gridDim.x) {
    const bool more = tile < ntiles;                                 // block-uniform
    if (more) {
      const long long t = tile * NT + tid;
      const bool live = t < total;
      const PhaseAVoxel v = glcm_phaseA_load<NT>(lev, centers, P, z0, out_z0, t, live, w);
      if (v.full) {
        glcm_phaseA_voxel<true, NT>(w, eq, T, P, v, true, out, fstride, queue, qcount);
      } else if (v.center) {
        defer[atomicAdd(&ndefer, 1u)] = (unsigned)t;
      } else if (live) {
#pragma unroll
        for (int k = 0; k < GLCM_NF; k++) out[k * fstride + v.oi] = P.init_value;
      }
    }
    __syncthreads();
    const unsigned nd = ndefer;
    __syncthreads();
    // the general body over the last `count` list entries (idle threads run on an all-zero window)
    const unsigned count = more ? (nd >= NT ? NT : 0) : nd;
    if (count) {
      if (tid == 0) ndefer = nd - count;
      const bool dlive = (unsigned)tid < count;
      const PhaseAVoxel v = glcm_phaseA_load<NT>(lev, centers, P, z0, out_z0, dlive ? defer[nd - count + tid] : 0, dlive, w);
      glcm_phaseA_voxel<false, NT>(w, eq, T, P, v, dlive, out, fstride, queue, qcount);
      __syncthreads();                                               // every entry read before the list grows again
    }
    if (!more) break;
  }
}


__global__ void __launch_bounds__(256)
glcm_fast_finish_kernel(const __grid_constant__ VoxParams P, const GlcmTask* __restrict__ queue,
                        const unsigned* __restrict__ qcount, const double* __restrict__ res,
                        double* __restrict__ mcc_map /* out + G_MCC*fstride */, int out_z0) {
  const unsigned n = *qcount;
  const long long plane = (long long)P.Y * P.X;
  for (unsigned k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const GlcmTask e = queue[k];
    if (!e.count) continue;
    double add = 0;
    for (int j = 0; j < e.count; j++) add += res[k + j];
    const int z = (int)(e.vi / P.sz);
    const long long oi = e.vi - (long long)out_z0 * plane;   // contiguous volume: vi = z*plane + rem
    (void)z;
    mcc_map[oi] += add / e.n_ok;
  }
}

}  // namespace rb
