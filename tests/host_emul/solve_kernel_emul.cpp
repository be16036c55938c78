// TEST-ONLY: the CUDA execution model of ONE thread block on the CPU, to run the text of
// pyradiomics_b200/csrc/glcm_kernels.cuh (tile counting sort, size groups, block-uniform dense solves
// with barriers, the register Lanczos with its per-thread shared-memory vectors) without a GPU: one std::thread per CUDA
// thread, __syncthreads() = pthread barrier, __shared__ = static storage (blocks run one at a time),
// atomics = GCC atomics.  Built with -fsanitize=thread the same run is a data-race check of the
// kernel's shared-memory protocol.
//
//   g++ -O1 -g -std=c++17 -pthread [-fsanitize=thread] -shared -fPIC solve_kernel_emul.cpp
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <string.h>

#include <atomic>
#include <thread>
#include <vector>

#define RB_EMULATE_BLOCK 1
#define __global__
#define __shared__ static
#define __restrict__
#define __launch_bounds__(...)
#define __grid_constant__
#define __device__
#define __forceinline__ inline
struct EmuDim { unsigned x, y, z; };
static thread_local EmuDim threadIdx;
static EmuDim blockIdx, blockDim, gridDim;
static pthread_barrier_t g_barrier;
static std::atomic<int> g_or_acc{0};
static inline void __syncthreads() { pthread_barrier_wait(&g_barrier); }
static inline int __syncthreads_or(int p) {
  if (p) g_or_acc.store(1, std::memory_order_relaxed);
  pthread_barrier_wait(&g_barrier);
  const int r = g_or_acc.load(std::memory_order_relaxed);
  pthread_barrier_wait(&g_barrier);
  if (threadIdx.x == 0) g_or_acc.store(0, std::memory_order_relaxed);
  pthread_barrier_wait(&g_barrier);
  return r;
}
static inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __ffs(int x) { return __builtin_ffs(x); }
#define RB_GLCM_BLOCK_SYNC 1
static double* g_dyn_shared = nullptr;
#define RB_DYN_SHARED(type, name) type* name = (type*)g_dyn_shared

#include "../../pyradiomics_b200/csrc/host_common.hpp"
#include "../../pyradiomics_b200/csrc/glcm_kernels.cuh"

using namespace rb;

template <int KIND>
static void run_kind(const uint8_t* lev, const VoxParams& P, const GlcmFastTables* T, const GlcmTask* q, unsigned n,
                     double* res, int nblocks) {
  const unsigned cnt = n;
  blockDim = {128, 1, 1};
  gridDim = {(unsigned)nblocks, 1, 1};
  std::vector<double> dyn((size_t)LZ_NARR * 18 * 128, 1e300);
  g_dyn_shared = dyn.data();
  for (int b = 0; b < nblocks; b++) {
    blockIdx = {(unsigned)b, 0, 0};
    pthread_barrier_init(&g_barrier, nullptr, 128);
    std::vector<std::thread> th;
    for (unsigned t = 0; t < 128; t++)
      th.emplace_back([=, &cnt]() {
        threadIdx = {t, 0, 0};
        glcm_fast_solve_kernel<KIND>(lev, P, T, q, &cnt, res, 0);
      });
    for (auto& x : th) x.join();
    pthread_barrier_destroy(&g_barrier);
  }
}

// lev: uint8 [Z][Y][X]; tasks from phase A of every voxel; res_kernel: results through the emulated kernels;
// res_direct: the same tasks through glcm_fast_solve<-1> one by one.  Returns the number of tasks (<= cap).
extern "C" int emul_solve_kernels(const uint8_t* lev, int Z, int Y, int X, int Ng, int nblocks, int cap, double* res_kernel,
                                  double* res_direct, int* cls_out) {
  VoxSettings s;
  memset(&s, 0, sizeof(s));
  s.Ng = Ng; s.n_roi_levels = Ng; s.kernelRadius = 1; s.ndist = 1; s.distances[0] = 1; s.symmetricalGLCM = 1;
  VoxParams P;
  if (fill_vox_params(C_GLCM, Z, Y, X, s, P)) return -1;              // (marks every angle alive)
  GlcmFastTables* T = new GlcmFastTables;
  glcm_fast_build_tables(*T, Ng);
  GlcmSolveTables ST;
  glcm_solve_tables_from(*T, ST);
  std::vector<GlcmTask> q;
  pthread_barrier_init(&g_barrier, nullptr, 1);       // phase A is called from this single thread: its barriers are 1-party
  for (int z = 0; z < Z; z++) for (int y = 0; y < Y; y++) for (int x = 0; x < X; x++) {
    const long long vi = ((long long)z * Y + y) * X + x;
    if (!lev[vi]) continue;
    uint8_t w[27]; int p = 0;
    for (int dz = -1; dz <= 1; dz++) for (int dy = -1; dy <= 1; dy++) for (int dx = -1; dx <= 1; dx++, p++) {
      const int zz = z + dz, yy = y + dy, xx = x + dx;
      w[p] = (zz >= 0 && zz < Z && yy >= 0 && yy < Y && xx >= 0 && xx < X) ? lev[vi + ((long long)dz * Y + dy) * X + dx] : 0;
    }
    uint32_t eq[27]; double f[GLCM_NF]; int n_ok = 0; unsigned long long tcls = 0;
    const uint32_t tasks = glcm_fast_voxel_phaseA(w, 1, eq, 1, *T, P, f, &n_ok, &tcls);
    for (int sl = 0; sl < GF_NA; sl++) if (tasks >> sl & 1u) {
      GlcmTask e; e.vi = vi; e.slot = (uint8_t)sl; e.n_ok = (uint8_t)n_ok; e.count = 0;
      e.cls = (uint8_t)(tcls >> (GF_CLS_BITS * sl) & (GF_NCLS - 1)); e.unused = 0.f;
      if ((int)q.size() < cap) {
        res_direct[q.size()] = glcm_fast_solve(w, 1, ST, sl, e.cls);
        cls_out[q.size()] = e.cls;
        q.push_back(e);
      }
    }
  }
  pthread_barrier_destroy(&g_barrier);
  const unsigned n = (unsigned)q.size();
  for (unsigned k = 0; k < n; k++) res_kernel[k] = -12345.0;      // a task no kernel picks up stays visible
  run_kind<0>(lev, P, T, q.data(), n, res_kernel, nblocks);
  run_kind<1>(lev, P, T, q.data(), n, res_kernel, nblocks);
  run_kind<2>(lev, P, T, q.data(), n, res_kernel, nblocks);
  delete T;
  return (int)n;
}


// one emulated launch: `nblocks` blocks of `nthreads` threads, run one block after another
template <class F>
static void emu_launch(int nblocks, int nthreads, F body) {
  blockDim = {(unsigned)nthreads, 1, 1};
  gridDim = {(unsigned)nblocks, 1, 1};
  for (int b = 0; b < nblocks; b++) {
    blockIdx = {(unsigned)b, 0, 0};
    pthread_barrier_init(&g_barrier, nullptr, nthreads);
    std::vector<std::thread> th;
    for (unsigned t = 0; t < (unsigned)nthreads; t++)
      th.emplace_back([=]() { threadIdx = {t, 0, 0}; body(); });
    for (auto& x : th) x.join();
    pthread_barrier_destroy(&g_barrier);
  }
}

// The whole fused GLCM path of glcm_fast_run on the CPU: phase A (256-thread blocks, per-angle barriers, queue
// reservation by atomics), the three solve kernels, the finish kernel; planes [0, Z) in chunks of `zchunk`.
// out: [24][Z][Y][X] float64.  Returns the total number of eigen-tasks.
extern "C" long long emul_glcm_pipeline(const uint8_t* lev, int Z, int Y, int X, int Ng, int zchunk, double* out) {
  VoxSettings s;
  memset(&s, 0, sizeof(s));
  s.Ng = Ng; s.n_roi_levels = Ng; s.kernelRadius = 1; s.ndist = 1; s.distances[0] = 1; s.symmetricalGLCM = 1;
  VoxParams P;
  if (fill_vox_params(C_GLCM, Z, Y, X, s, P)) return -1;
  GlcmFastTables* T = new GlcmFastTables;
  glcm_fast_build_tables(*T, Ng);
  const long long plane = (long long)Y * X, fstride = (long long)Z * plane;
  std::vector<GlcmTask> q((size_t)zchunk * plane * GF_NA);
  std::vector<double> res(q.size());
  std::vector<double> dyn((size_t)LZ_NARR * 18 * 128, 1e300);
  g_dyn_shared = dyn.data();
  long long total_tasks = 0;
  for (int za = 0; za < Z; za += zchunk) {
    const int zb = za + zchunk < Z ? za + zchunk : Z;
    unsigned count = 0;
    GlcmTask* qp = q.data(); double* rp = res.data(); unsigned* cp = &count;
    emu_launch(3, 256, [=]() { glcm_fast_kernel<1, 256>(lev, nullptr, P, T, out, fstride, za, zb, 0, qp, cp); });
    for (unsigned k = 0; k < count; k++) res[k] = -12345.0;
    // one launch per size group of the n <= 8 and Lanczos kinds and one for the whole n <= 12 kind: glcm_fast_run
    // splits the dense kinds the other way round, so between them both paths of `only` run for both dense kinds
    for (int g = 4; g <= 8; g += 2) emu_launch(2, 128, [=]() { glcm_fast_solve_kernel<0>(lev, P, T, qp, cp, rp, g); });
    emu_launch(2, 128, [=]() { glcm_fast_solve_kernel<1>(lev, P, T, qp, cp, rp, 0); });
    for (int g = 18; g >= 14; g -= 2) emu_launch(2, 128, [=]() { glcm_fast_solve_kernel<2>(lev, P, T, qp, cp, rp, g); });
    emu_launch(2, 256, [=]() { glcm_fast_finish_kernel(P, qp, cp, rp, out + (long long)G_MCC * fstride, 0); });
    total_tasks += count;
  }
  delete T;
  return total_tasks;
}
