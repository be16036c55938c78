// Segment-based texture matrices of ONE ROI from a device-resident packed level volume (reference
// radiomics/src/cmatrices.c: calculate_glcm :4-92, calculate_gldm :660-754, calculate_ngtdm :543-658, calculate_glrlm
// :299-541).
//
//   segment_matrices       GLCM + GLDM + NGTDM in one pass, by one of two kernels with the same flags and accumulators:
//     seg_tile_kernel      8-bit levels, offsets up to 3 and histograms that fit shared memory: a CTA stages a
//                          (TZ+2H) x (TY+2H) x 96-byte box of the level volume in shared memory -- by TMA
//                          (cp.async.bulk.tensor.3d, out-of-volume coordinates are zero-filled by the hardware =
//                          "unmasked", double-buffered on an mbarrier) when the row pitch allows a tensor map, else by
//                          cooperative loads -- walks the 13 / 26 offsets in shared memory and accumulates into per-CTA
//                          shared-memory histograms (GLCM Ng x Ng x Na when it fits), flushed once per CTA with
//                          coalesced atomics.
//     seg_direct_kernel    everything else (16-bit levels, longer offsets, more levels): one thread per voxel, global
//                          loads, the GLCM histogram privatised in shared memory when it fits.
//   segment_glrlm          seg_glrlm_ends_kernel: every voxel that ENDS a run (successor outside / unmasked / another
//                          level) walks back to the run's start: all voxels work, loads coalesce along x.  The
//                          reference's "angle without a line of two voxels loses its length-1 column" rule
//                          (cmatrices.c:524-534) comes from a pigeonhole count: some line holds two masked voxels <=>
//                          #masked voxels > #lines that hold any.
//   segment_glszm          GLSZM's zones (cmatrices.c:94-279): union-find connected-component labelling (26 / 8
//                          neighbours of equal level) -> zone sizes -> one (gray, size) pair per zone.
// Integer counts are exact; NGTDM's s_i is accumulated as integers T[g][count] += |g*count - sum| and divided by count
// once at the end, so both kernels give bit-identical matrices.
//
// Every builder starts from segment_geometry and runs all its launches and copies on the caller's stream.
#include <cuda.h>

#include <vector>

#include "common.cuh"
#include "host_common.hpp"
#include "vox_features.cuh"

namespace rb {

struct SegAngles {
  int na;                 // unidirectional offsets (GLCM); GLDM / NGTDM use +- each of them
  int8_t a[NW_MAX][3];
  explicit SegAngles(const AngleSet& A) : na(A.na) { memcpy(a, A.a, sizeof(a[0]) * na); }
};
struct SegVol {
  int Z, Y, X;
  long long pitch_y, pitch_z;      // element strides (x stride 1)
};

constexpr int ST_TX = 64, ST_THREADS = 256;
// The staged box starts ST_XOFF columns left of the tile: TMA wants the innermost start coordinate 16-byte aligned (a box
// at x0-1 faults with "illegal instruction", at x0-16 it loads and zero-fills), and tiles start at multiples of 64.
constexpr int ST_XOFF = 16, ST_BX = ST_XOFF + ST_TX + 16;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%1], %0;" ::"r"(count), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%1], %0;" ::"r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  asm volatile(
      "{\n\t.reg .pred P1;\n\tLAB_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\tbra LAB_WAIT;\n\tDONE:\n\t}" ::"r"(smem_u32(bar)), "r"(phase) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"((uint64_t)map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}

struct SegTileGeom {
  int tz, ty;            // tile = tz x ty x ST_TX voxels (tz * ty * ST_TX = 8 * ST_THREADS)
  int H;                 // halo = largest offset component
  int bx, by, bz;        // staged box: bx = ST_BX bytes per row (16-byte aligned start), by = ty + 2H rows, bz = tz + 2H planes
  int ntx, nty, ntz;     // tiles per axis
  int glcm_shared;       // GLCM histogram lives in shared memory
};

// flags: 1 = GLCM, 2 = GLDM, 4 = NGTDM
template <bool TMA>
__global__ void __launch_bounds__(ST_THREADS)
seg_tile_kernel(const uint8_t* __restrict__ lev, SegVol V, const __grid_constant__ SegAngles A, const SegTileGeom G, int Ng,
                int alpha, int flags, const __grid_constant__ CUtensorMap tmap, unsigned* __restrict__ glcm_hist,
                unsigned* __restrict__ gldm_hist, unsigned long long* __restrict__ ngtdm_acc) {
  extern __shared__ __align__(128) uint8_t seg_smem[];
  const int box = G.bx * G.by * G.bz, box_al = (box + 127) & ~127;
  uint8_t* tile0 = seg_smem;                                   // two staged boxes
  unsigned long long* s_ng = reinterpret_cast<unsigned long long*>(seg_smem + 2 * box_al);      // [Ng][2na+2]
  const int ng_cols = 2 * A.na + 2, gd_cols = 2 * (2 * A.na) + 1;
  unsigned* s_gd = reinterpret_cast<unsigned*>(s_ng + (size_t)((flags & 4) ? Ng * ng_cols : 0));     // [Ng][2*Na_bi+1]
  unsigned* s_gl = s_gd + (size_t)((flags & 2) ? Ng * gd_cols : 0);                                   // [Ng][Ng][na]
  __shared__ uint64_t bar[2];
  const int tid = threadIdx.x;
  const int n_gl = (flags & 1) && G.glcm_shared ? Ng * Ng * A.na : 0;
  for (int i = tid; i < n_gl; i += ST_THREADS) s_gl[i] = 0;
  if (flags & 2) for (int i = tid; i < Ng * gd_cols; i += ST_THREADS) s_gd[i] = 0;
  if (flags & 4) for (int i = tid; i < Ng * ng_cols; i += ST_THREADS) s_ng[i] = 0;
  if (TMA && tid == 0) {
    mbar_init(&bar[0], 1); mbar_init(&bar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int ntiles = G.ntx * G.nty * G.ntz;
  const int H = G.H;
  auto origin = [&](int t, int& x0, int& y0, int& z0) {
    x0 = (t % G.ntx) * ST_TX; y0 = (t / G.ntx % G.nty) * G.ty; z0 = (t / (G.ntx * G.nty)) * G.tz;
  };
  auto stage = [&](int t, int buf) {                // box with origin (x0-H, y0-H, z0-H); zeros outside the volume
    int x0, y0, z0;
    origin(t, x0, y0, z0);
    uint8_t* dst = tile0 + buf * box_al;
    if (TMA) {
      if (tid == 0) {
        mbar_expect_tx(&bar[buf], (uint32_t)box);
        tma_load_3d(dst, &tmap, &bar[buf], x0 - ST_XOFF, y0 - H, z0 - H);
      }
    } else {
      for (int i = tid; i < box; i += ST_THREADS) {
        const int c = i % G.bx, r = i / G.bx % G.by, p = i / (G.bx * G.by);
        const int x = x0 - ST_XOFF + c, y = y0 - H + r, z = z0 - H + p;
        dst[i] = (x >= 0 && x < V.X && y >= 0 && y < V.Y && z >= 0 && z < V.Z) ? lev[(long long)z * V.pitch_z + (long long)y * V.pitch_y + x]
                                                                               : (uint8_t)0;
      }
    }
  };
  int it = 0;
  if ((int)blockIdx.x < ntiles) stage(blockIdx.x, 0);
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x, it++) {
    const int buf = it & 1;
    const int tn = t + gridDim.x;
    if (TMA) {
      if (tn < ntiles) stage(tn, buf ^ 1);          // prefetch the next box while this one is consumed
      mbar_wait(&bar[buf], (uint32_t)(it >> 1) & 1u);
    } else {
      __syncthreads();                               // the cooperative stores of this box are visible
    }
    const uint8_t* tl = tile0 + buf * box_al;
    int x0, y0, z0;
    origin(t, x0, y0, z0);
#pragma unroll 1
    for (int k = 0; k < 8; k++) {
      const int v = k * ST_THREADS + tid;           // voxel of the tile: x fastest
      const int lx = v % ST_TX, ly = v / ST_TX % G.ty, lz = v / (ST_TX * G.ty);
      if (x0 + lx >= V.X || y0 + ly >= V.Y || z0 + lz >= V.Z) continue;
      const int c = ((lz + H) * G.by + (ly + H)) * G.bx + (lx + ST_XOFF);
      const int gi = tl[c];
      if (!gi) continue;
      int dep = 0, cnt = 0, sum = 0;
      for (int a = 0; a < A.na; a++) {
        const int off = (A.a[a][0] * G.by + A.a[a][1]) * G.bx + A.a[a][2];
        const int gj = tl[c + off], gr = tl[c - off];
        if ((flags & 1) && gj) {
          const int b = ((gi - 1) * Ng + (gj - 1)) * A.na + a;
          if (G.glcm_shared) atomicAdd(&s_gl[b], 1u); else atomicAdd(&glcm_hist[b], 1u);
        }
        if (gj) { cnt++; sum += gj; const int d = gi > gj ? gi - gj : gj - gi; dep += d <= alpha; }
        if (gr) { cnt++; sum += gr; const int d = gi > gr ? gi - gr : gr - gi; dep += d <= alpha; }
      }
      if (flags & 2) atomicAdd(&s_gd[(gi - 1) * gd_cols + dep], 1u);
      if (flags & 4) {
        atomicAdd(&s_ng[(gi - 1) * ng_cols], 1ull);
        if (cnt) {
          long long num = (long long)gi * cnt - sum;
          if (num < 0) num = -num;
          if (num) atomicAdd(&s_ng[(gi - 1) * ng_cols + 1 + cnt], (unsigned long long)num);
        }
      }
    }
    __syncthreads();                                 // everyone is done with this box (it is restaged two tiles later)
    if (!TMA && tn < ntiles) stage(tn, buf ^ 1);
  }
  __syncthreads();
  for (int i = tid; i < n_gl; i += ST_THREADS) if (s_gl[i]) atomicAdd(&glcm_hist[i], s_gl[i]);
  if (flags & 2) for (int i = tid; i < Ng * gd_cols; i += ST_THREADS) if (s_gd[i]) atomicAdd(&gldm_hist[i], s_gd[i]);
  if (flags & 4) for (int i = tid; i < Ng * ng_cols; i += ST_THREADS) if (s_ng[i]) atomicAdd(&ngtdm_acc[i], s_ng[i]);
}

// Same flags and accumulator layouts as seg_tile_kernel (A = the unidirectional offsets; GLDM / NGTDM also use their
// mirrors).  The GLCM histogram lives in shared memory when glcm_shared.
template <typename T>
__global__ void __launch_bounds__(256)
seg_direct_kernel(const T* __restrict__ lev, SegVol V, const __grid_constant__ AngleSet A, int Ng, int alpha, int flags,
                  int glcm_shared, unsigned* __restrict__ glcm_hist, unsigned* __restrict__ gldm_hist,
                  unsigned long long* __restrict__ ngtdm_acc) {
  extern __shared__ unsigned s_glcm[];
  const int n_gl = glcm_shared ? Ng * Ng * A.na : 0;
  for (int i = threadIdx.x; i < n_gl; i += blockDim.x) s_glcm[i] = 0;
  __syncthreads();
  unsigned* gl = glcm_shared ? s_glcm : glcm_hist;
  const int ng_cols = 2 * A.na + 2, gd_cols = 2 * (2 * A.na) + 1;
  const long long n = (long long)V.Z * V.Y * V.X, plane = (long long)V.Y * V.X;
  auto in = [&](int z, int y, int x) { return z >= 0 && z < V.Z && y >= 0 && y < V.Y && x >= 0 && x < V.X; };
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const int gi = lev[t];
    if (!gi) continue;
    const int z = (int)(t / plane), rem = (int)(t % plane), y = rem / V.X, x = rem % V.X;
    int dep = 0, cnt = 0, sum = 0;
    for (int a = 0; a < A.na; a++) {
      const int dz = A.a[a][0], dy = A.a[a][1], dx = A.a[a][2];
      const long long off = dz * V.pitch_z + dy * V.pitch_y + dx;
      const int gj = in(z + dz, y + dy, x + dx) ? lev[t + off] : 0;
      if ((flags & 1) && gj) atomicAdd(&gl[((size_t)(gi - 1) * Ng + (gj - 1)) * A.na + a], 1u);
      if (flags & 6) {
        const int gr = in(z - dz, y - dy, x - dx) ? lev[t - off] : 0;
        if (gj) { cnt++; sum += gj; const int d = gi > gj ? gi - gj : gj - gi; dep += d <= alpha; }
        if (gr) { cnt++; sum += gr; const int d = gi > gr ? gi - gr : gr - gi; dep += d <= alpha; }
      }
    }
    if (flags & 2) atomicAdd(&gldm_hist[(gi - 1) * gd_cols + dep], 1u);
    if (flags & 4) {
      atomicAdd(&ngtdm_acc[(gi - 1) * ng_cols], 1ull);
      if (cnt) {
        long long num = (long long)gi * cnt - sum;
        if (num < 0) num = -num;
        if (num) atomicAdd(&ngtdm_acc[(gi - 1) * ng_cols + 1 + cnt], (unsigned long long)num);
      }
    }
  }
  if (glcm_shared) {
    __syncthreads();
    for (int i = threadIdx.x; i < n_gl; i += blockDim.x) if (s_glcm[i]) atomicAdd(&glcm_hist[i], s_glcm[i]);
  }
}

// ---- GLRLM by run ends ----------------------------------------------------------------------------------------------
// hist[((g-1)*Nr + len-1)*na + a]; short runs (len <= RL_SH) of every (level, angle) are counted in shared memory first.
constexpr int RL_SH = 4;
template <typename T>
__global__ void __launch_bounds__(256)
seg_glrlm_ends_kernel(const T* __restrict__ lev, SegVol V, const __grid_constant__ SegAngles A, int Ng, int Nr,
                      unsigned* __restrict__ hist, unsigned long long* __restrict__ counts /* [0]=masked voxels, [1+a]=lines holding a voxel */,
                      int* __restrict__ status) {
  extern __shared__ unsigned s_rl[];                 // [Ng][RL_SH][na] when it fits (sh_ok), else unused
  __shared__ unsigned s_lines[NW_MAX];
  __shared__ unsigned s_masked;
  const int na = A.na;
  const bool sh_ok = (size_t)Ng * RL_SH * na * 4 <= 96 * 1024;
  if (sh_ok) for (int i = threadIdx.x; i < Ng * RL_SH * na; i += blockDim.x) s_rl[i] = 0;
  for (int i = threadIdx.x; i < na; i += blockDim.x) s_lines[i] = 0;
  if (threadIdx.x == 0) s_masked = 0;
  __syncthreads();
  const long long n = (long long)V.Z * V.Y * V.X, plane = (long long)V.Y * V.X;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const int z = (int)(t / plane), rem = (int)(t % plane), y = rem / V.X, x = rem % V.X;
    const long long vi = (long long)z * V.pitch_z + (long long)y * V.pitch_y + x;
    const int g = lev[vi];
    if (!g) continue;
    atomicAdd(&s_masked, 1u);
    for (int a = 0; a < na; a++) {
      const int az = A.a[a][0], ay = A.a[a][1], ax = A.a[a][2];
      const long long step = (long long)az * V.pitch_z + (long long)ay * V.pitch_y + ax;
      // am I the first masked voxel of my line?  (walk back over unmasked voxels: rare inside a blob-shaped ROI)
      {
        int pz = z - az, py = y - ay, px = x - ax;
        long long pi = vi - step;
        bool first = true;
        while (pz >= 0 && pz < V.Z && py >= 0 && py < V.Y && px >= 0 && px < V.X) {
          if (lev[pi]) { first = false; break; }
          pz -= az; py -= ay; px -= ax; pi -= step;
        }
        if (first) atomicAdd(&s_lines[a], 1u);
      }
      // run end?
      const int nz = z + az, ny = y + ay, nx = x + ax;
      const bool has_next = nz >= 0 && nz < V.Z && ny >= 0 && ny < V.Y && nx >= 0 && nx < V.X;
      if (has_next && lev[vi + step] == g) continue;
      int len = 1;
      {
        int pz = z - az, py = y - ay, px = x - ax;
        long long pi = vi - step;
        while (pz >= 0 && pz < V.Z && py >= 0 && py < V.Y && px >= 0 && px < V.X && lev[pi] == g) {
          len++; pz -= az; py -= ay; px -= ax; pi -= step;
        }
      }
      if (len > Nr) { atomicOr(status, 1); continue; }
      if (sh_ok && len <= RL_SH) atomicAdd(&s_rl[((g - 1) * RL_SH + (len - 1)) * na + a], 1u);
      else atomicAdd(&hist[((size_t)(g - 1) * Nr + (len - 1)) * na + a], 1u);
    }
  }
  __syncthreads();
  if (sh_ok)
    for (int i = threadIdx.x; i < Ng * RL_SH * na; i += blockDim.x)
      if (s_rl[i]) {
        const int a = i % na, l = i / na % RL_SH, g = i / (na * RL_SH);
        if (l < Nr) atomicAdd(&hist[((size_t)g * Nr + l) * na + a], s_rl[i]);
      }
  for (int i = threadIdx.x; i < na; i += blockDim.x) if (s_lines[i]) atomicAdd(&counts[1 + i], (unsigned long long)s_lines[i]);
  if (threadIdx.x == 0 && s_masked) atomicAdd(&counts[0], (unsigned long long)s_masked);
}

// ---- GLSZM: union-find connected components over equal-level 26/8-neighbours -----------------------------------------
struct Vol {
  int Z, Y, X;
  __host__ __device__ long long n() const { return (long long)Z * Y * X; }
  __device__ bool in(int z, int y, int x) const { return z >= 0 && z < Z && y >= 0 && y < Y && x >= 0 && x < X; }
  __device__ long long idx(int z, int y, int x) const { return ((long long)z * Y + y) * X + x; }
};

__device__ __forceinline__ int uf_find(int* L, int i) {
  int p = L[i];
  while (p != i) { i = p; p = L[i]; }
  return i;
}
__device__ __forceinline__ void uf_union(int* L, int a, int b) {
  while (true) {
    a = uf_find(L, a); b = uf_find(L, b);
    if (a == b) return;
    if (a < b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(&L[a], b);
    if (old == a) return;
    a = old;
  }
}

template <typename T>
__global__ void __launch_bounds__(256) ccl_init_kernel(const T* __restrict__ lev, long long n, int* __restrict__ L) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    L[i] = lev[i] ? (int)i : -1;
}
template <typename T>
__global__ void __launch_bounds__(256)
ccl_merge_kernel(const T* __restrict__ lev, Vol V, const __grid_constant__ AngleSet A, int* __restrict__ L) {
  const long long n = V.n(), plane = (long long)V.Y * V.X;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const int g = lev[t];
    if (!g) continue;
    const int z = (int)(t / plane), rem = (int)(t % plane), y = rem / V.X, x = rem % V.X;
    for (int a = 0; a < A.na; a++) {       // unidirectional half of the neighbourhood is enough
      const int z2 = z + A.a[a][0], y2 = y + A.a[a][1], x2 = x + A.a[a][2];
      if (!V.in(z2, y2, x2)) continue;
      const long long j = V.idx(z2, y2, x2);
      if (lev[j] == g) uf_union(L, (int)t, (int)j);
    }
  }
}
__global__ void __launch_bounds__(256) ccl_count_kernel(int* __restrict__ L, long long n, unsigned* __restrict__ size) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (L[i] < 0) continue;
    const int r = uf_find(L, (int)i);
    atomicAdd(&size[r], 1u);
  }
}
template <typename T>
__global__ void __launch_bounds__(256)
ccl_zones_kernel(const T* __restrict__ lev, const int* __restrict__ L, const unsigned* __restrict__ size, long long n,
                 int* __restrict__ zones, unsigned* __restrict__ nzones, unsigned* __restrict__ max_region) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (L[i] != (int)i) continue;            // roots only
    const unsigned k = atomicAdd(nzones, 1u);
    zones[2 * (size_t)k] = lev[i];
    zones[2 * (size_t)k + 1] = (int)size[i];
    atomicMax(max_region, size[i]);
  }
}

// counts -> float64 with the multi-voxel-line rule (cmatrices.c:524-534) from the pigeonhole counts
__global__ void glrlm_to_f64_kernel(const unsigned* __restrict__ hist, long long n, double* __restrict__ out,
                                    const unsigned long long* __restrict__ counts, int Nr, int na) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int a = (int)(i % na), r = (int)((i / na) % Nr);
    const bool multi = counts[0] > counts[1 + a];
    out[i] = (r == 0 && !multi) ? 0.0 : (double)hist[i];
  }
}
__global__ void u32_to_f64_kernel(const unsigned* __restrict__ hist, long long n, double* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) out[i] = (double)hist[i];
}
__global__ void ngtdm_seg_finish_kernel(const unsigned long long* __restrict__ acc, int Ng, int ncnt, double* __restrict__ out) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= Ng) return;
  const int ncol = ncnt + 2;
  double s = 0;
  for (int c = 1; c <= ncnt; c++) s += (double)acc[g * ncol + 1 + c] / (double)c;
  out[g * 3 + 0] = (double)acc[g * ncol];
  out[g * 3 + 1] = s;
  out[g * 3 + 2] = (double)(g + 1);
}

int segment_geometry(const int* size, int nd, const int* distances, int ndist, bool bidirectional, int force2D,
                     int force2Ddimension, int Ng, int na_max, int* angles_out, SegmentGeometry& G) {
  G.Z = nd == 3 ? size[0] : 1; G.Y = size[nd - 2]; G.X = size[nd - 1];
  G.n = (long long)G.Z * G.Y * G.X;
  if (Ng < 1 || Ng > 65535) return fail(RB_ERR_UNSUPPORTED, "Ng=%d outside 1..65535", Ng);
  if (G.n <= 0 || G.n >= (1ll << 31)) return fail(RB_ERR_UNSUPPORTED, "volume must have 1..2^31-1 voxels");
  std::vector<int> ang;
  const int na = generate_angles(size, nd, distances, ndist, bidirectional, force2D ? force2Ddimension : -1, ang);
  if (na <= 0) return fail(RB_ERR_ARG, "Error getting angle count.");
  if (na > na_max) return fail(RB_ERR_UNSUPPORTED, "more than %d angles", NA_MAX);
  G.A.na = na;
  G.H = 0;
  for (int a = 0; a < na; a++)
    for (int d = 0; d < 3; d++) {
      const int v = d < 3 - nd ? 0 : ang[a * nd + d - (3 - nd)];
      G.A.a[a][d] = (int8_t)v;
      G.H = v > G.H ? v : (-v > G.H ? -v : G.H);
    }
  if (angles_out) memcpy(angles_out, ang.data(), sizeof(int) * ang.size());
  return RB_OK;
}

// B200_SEG_TMA=0 forces the cooperative-load staging (A/B runs, tests); default: TMA whenever a tensor map can be built
static bool seg_tma_enabled() {
  const char* e = getenv("B200_SEG_TMA");
  return !(e && e[0] == '0');
}

// seg_tile_kernel's plan for a volume, or 0 when its shared memory would exceed 220 KB
static size_t tile_plan(int Z, int Y, int X, int H, int Ng, int na, int flags, SegTileGeom& G) {
  G.H = H;
  if (Z == 1) { G.tz = 1; G.ty = 32; } else { G.tz = 4; G.ty = 8; }
  G.bx = ST_BX; G.by = G.ty + 2 * H; G.bz = G.tz + 2 * H;
  G.ntx = (X + ST_TX - 1) / ST_TX; G.nty = (Y + G.ty - 1) / G.ty; G.ntz = (Z + G.tz - 1) / G.tz;
  const int box_al = (G.bx * G.by * G.bz + 127) & ~127;
  const size_t n_gl = (size_t)Ng * Ng * na, n_gd = (size_t)Ng * (2 * (2 * na) + 1), n_ng = (size_t)Ng * (2 * na + 2);
  size_t smem = 2 * (size_t)box_al + ((flags & 4) ? n_ng * 8 : 0) + ((flags & 2) ? n_gd * 4 : 0);
  G.glcm_shared = (flags & 1) && smem + n_gl * 4 <= 200 * 1024;
  if (G.glcm_shared) smem += n_gl * 4;
  return smem > 220 * 1024 ? 0 : smem;
}

static int launch_tile(const uint8_t* lev, SegVol V, const AngleSet& A, const SegTileGeom& G, size_t smem, int Ng, int alpha,
                       int flags, unsigned* d_gl, unsigned* d_gd, unsigned long long* d_ng, cudaStream_t st) {
  const SegAngles S(A);
  // tensor map: needs a 16-byte aligned base and row / plane pitches that are multiples of 16 bytes
  CUtensorMap tmap;
  memset(&tmap, 0, sizeof tmap);
  bool tma = seg_tma_enabled() && (V.X % 16 == 0) && (((uintptr_t)lev & 15) == 0);
  if (tma) {
    const cuuint64_t gdim[3] = {(cuuint64_t)V.X, (cuuint64_t)V.Y, (cuuint64_t)V.Z};
    const cuuint64_t gstr[2] = {(cuuint64_t)V.X, (cuuint64_t)V.X * (cuuint64_t)V.Y};
    const cuuint32_t bdim[3] = {(cuuint32_t)G.bx, (cuuint32_t)G.by, (cuuint32_t)G.bz};
    const cuuint32_t estr[3] = {1, 1, 1};
    // the driver entry point is looked up at run time: the library must load on a box without libcuda (the CPU tests)
    typedef CUresult (*EncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static EncodeTiled encode = nullptr;
    static bool looked_up = false;
    if (!looked_up) {
      void* fn = nullptr;
      cudaDriverEntryPointQueryResult q;
      if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
        encode = (EncodeTiled)fn;
      looked_up = true;
    }
    const CUresult r = encode ? encode(&tmap, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, (void*)lev, gdim, gstr, bdim, estr,
                                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE)
                              : CUDA_ERROR_NOT_SUPPORTED;
    if (r != CUDA_SUCCESS) tma = false;              // (e.g. a plane pitch that is not a multiple of 16: fall back)
  }
  const int ntiles = G.ntx * G.nty * G.ntz;
  const int per_sm = smem > 110 * 1024 ? 1 : 2;
  int grid = sm_count() * per_sm;
  if (grid > ntiles) grid = ntiles;
  if (tma) {
    RB_CUDA(cudaFuncSetAttribute(seg_tile_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    seg_tile_kernel<true><<<grid, ST_THREADS, smem, st>>>(lev, V, S, G, Ng, alpha, flags, tmap, d_gl, d_gd, d_ng);
  } else {
    RB_CUDA(cudaFuncSetAttribute(seg_tile_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    seg_tile_kernel<false><<<grid, ST_THREADS, smem, st>>>(lev, V, S, G, Ng, alpha, flags, tmap, d_gl, d_gd, d_ng);
  }
  RB_LAUNCH_CHECK();
  return RB_OK;
}

template <typename T>
static int launch_direct(const T* lev, SegVol V, const AngleSet& A, int Ng, int alpha, int flags, unsigned* d_gl,
                         unsigned* d_gd, unsigned long long* d_ng, cudaStream_t st) {
  const long long n = (long long)V.Z * V.Y * V.X;
  const size_t sh = (size_t)Ng * Ng * A.na * 4;
  const int glcm_shared = (flags & 1) && sh <= 160 * 1024;
  if (glcm_shared) RB_CUDA(cudaFuncSetAttribute(seg_direct_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh));
  seg_direct_kernel<T><<<grid_for(n, 256, glcm_shared ? 1 : 8), 256, glcm_shared ? sh : 0, st>>>(lev, V, A, Ng, alpha, flags,
                                                                                             glcm_shared, d_gl, d_gd, d_ng);
  RB_LAUNCH_CHECK();
  return RB_OK;
}

// GLCM / GLDM / NGTDM of one packed level volume (uint8 or uint16) in one pass; outputs are HOST float64 buffers in the
// reference layouts (NULL = not wanted), angles_out gets the unidirectional offsets.  3-D volumes or 2-D (Z = 1).
int segment_matrices(const void* lev, int level_bytes, const int* size, int nd, const int* distances, int ndist, int Ng,
                     int alpha, int force2D, int force2Ddimension, double* glcm_host, double* gldm_host, double* ngtdm_host,
                     int* angles_out, cudaStream_t st) {
  SegmentGeometry sg;
  // GLCM counts the na offsets, GLDM / NGTDM each offset and its mirror
  int rc = segment_geometry(size, nd, distances, ndist, false, force2D, force2Ddimension, Ng,
                            (gldm_host || ngtdm_host) ? NA_MAX / 2 : NA_MAX, angles_out, sg);
  if (rc) return rc;
  const int flags = (glcm_host ? 1 : 0) | (gldm_host ? 2 : 0) | (ngtdm_host ? 4 : 0);
  if (!flags) return RB_OK;
  const AngleSet& A = sg.A;
  const int na = A.na;
  const size_t n_gl = (size_t)Ng * Ng * na, n_gd = (size_t)Ng * (2 * (2 * na) + 1), n_ng = (size_t)Ng * (2 * na + 2);
  DevBuf gl, gd, ng, out;
  if (flags & 1) { RB_CUDA(gl.alloc(n_gl * 4)); RB_CUDA(cudaMemsetAsync(gl.p, 0, n_gl * 4, st)); }
  if (flags & 2) { RB_CUDA(gd.alloc(n_gd * 4)); RB_CUDA(cudaMemsetAsync(gd.p, 0, n_gd * 4, st)); }
  if (flags & 4) { RB_CUDA(ng.alloc(n_ng * 8)); RB_CUDA(cudaMemsetAsync(ng.p, 0, n_ng * 8, st)); }
  // float64 staging for the largest requested matrix only: an unrequested GLCM at 16-bit Ng would be gigabytes
  size_t n_out = 3 * (size_t)Ng;
  if ((flags & 1) && n_gl > n_out) n_out = n_gl;
  if ((flags & 2) && n_gd > n_out) n_out = n_gd;
  RB_CUDA(out.alloc(n_out * 8));
  unsigned *d_gl = gl.as<unsigned>(), *d_gd = gd.as<unsigned>();
  unsigned long long* d_ng = ng.as<unsigned long long>();
  const SegVol V{sg.Z, sg.Y, sg.X, (long long)sg.X, (long long)sg.Y * sg.X};
  SegTileGeom G;
  const size_t smem = level_bytes == 1 && sg.H <= 3 && na <= NW_MAX ? tile_plan(sg.Z, sg.Y, sg.X, sg.H, Ng, na, flags, G) : 0;
  rc = smem ? launch_tile((const uint8_t*)lev, V, A, G, smem, Ng, alpha, flags, d_gl, d_gd, d_ng, st)
       : level_bytes == 1 ? launch_direct((const uint8_t*)lev, V, A, Ng, alpha, flags, d_gl, d_gd, d_ng, st)
                          : launch_direct((const uint16_t*)lev, V, A, Ng, alpha, flags, d_gl, d_gd, d_ng, st);
  if (rc) return rc;
  const int cg = sm_count() * 4;
  double* d_out = out.as<double>();
  if (flags & 1) {
    u32_to_f64_kernel<<<cg, 256, 0, st>>>(d_gl, (long long)n_gl, d_out);
    RB_CUDA(cudaMemcpyAsync(glcm_host, d_out, n_gl * 8, cudaMemcpyDeviceToHost, st));
    RB_CUDA(cudaStreamSynchronize(st));
  }
  if (flags & 2) {
    u32_to_f64_kernel<<<cg, 256, 0, st>>>(d_gd, (long long)n_gd, d_out);
    RB_CUDA(cudaMemcpyAsync(gldm_host, d_out, n_gd * 8, cudaMemcpyDeviceToHost, st));
    RB_CUDA(cudaStreamSynchronize(st));
  }
  if (flags & 4) {
    ngtdm_seg_finish_kernel<<<(Ng + 127) / 128, 128, 0, st>>>(d_ng, Ng, 2 * na, d_out);
    RB_CUDA(cudaMemcpyAsync(ngtdm_host, d_out, (size_t)Ng * 3 * 8, cudaMemcpyDeviceToHost, st));
    RB_CUDA(cudaStreamSynchronize(st));
  }
  return RB_OK;
}

// GLRLM of one packed level volume (uint8 or uint16) -> HOST float64 [Ng][Nr][Na]
int segment_glrlm(const void* lev, int level_bytes, const int* size, int nd, int Ng, int Nr, int force2D, int force2Ddimension,
                  double* glrlm_host, int* angles_out, cudaStream_t st) {
  SegmentGeometry sg;
  const int one[1] = {1};
  const int rc = segment_geometry(size, nd, one, 1, false, force2D, force2Ddimension, Ng, NW_MAX, angles_out, sg);
  if (rc) return rc;
  if (Nr < 1) return fail(RB_ERR_ARG, "Nr must be >= 1");
  const SegAngles A(sg.A);
  const int na = A.na;
  const size_t per = (size_t)Ng * Nr * na;
  DevBuf h, c, status, out;
  RB_CUDA(h.alloc(per * 4));
  RB_CUDA(c.alloc((1 + (size_t)na) * 8));
  RB_CUDA(status.alloc(4));
  RB_CUDA(out.alloc(per * 8));
  RB_CUDA(cudaMemsetAsync(h.p, 0, per * 4, st));
  RB_CUDA(cudaMemsetAsync(c.p, 0, (1 + (size_t)na) * 8, st));
  RB_CUDA(cudaMemsetAsync(status.p, 0, 4, st));
  unsigned* d_h = h.as<unsigned>();
  unsigned long long* d_c = c.as<unsigned long long>();
  int* d_st = status.as<int>();
  const SegVol V{sg.Z, sg.Y, sg.X, (long long)sg.X, (long long)sg.Y * sg.X};
  const int grid = grid_for(sg.n, 256, 8);
  const size_t sh = (size_t)Ng * RL_SH * na * 4 <= 96 * 1024 ? (size_t)Ng * RL_SH * na * 4 : 0;
  if (level_bytes == 1) {
    RB_CUDA(cudaFuncSetAttribute(seg_glrlm_ends_kernel<uint8_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    seg_glrlm_ends_kernel<uint8_t><<<grid, 256, sh, st>>>((const uint8_t*)lev, V, A, Ng, Nr, d_h, d_c, d_st);
  } else {
    RB_CUDA(cudaFuncSetAttribute(seg_glrlm_ends_kernel<uint16_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    seg_glrlm_ends_kernel<uint16_t><<<grid, 256, sh, st>>>((const uint16_t*)lev, V, A, Ng, Nr, d_h, d_c, d_st);
  }
  RB_LAUNCH_CHECK();
  glrlm_to_f64_kernel<<<sm_count() * 4, 256, 0, st>>>(d_h, (long long)per, out.as<double>(), d_c, Nr, na);
  RB_LAUNCH_CHECK();
  int stv = 0;
  RB_CUDA(cudaMemcpyAsync(&stv, d_st, 4, cudaMemcpyDeviceToHost, st));
  RB_CUDA(cudaMemcpyAsync(glrlm_host, out.p, per * 8, cudaMemcpyDeviceToHost, st));
  RB_CUDA(cudaStreamSynchronize(st));
  if (stv & 1) return fail(RB_ERR_LEVEL_RANGE, "Calculation of GLRLM Failed: run longer than Nr");
  return RB_OK;
}

// GLSZM phase one of a packed level volume (uint8 or uint16) into a new handle on `st` (one (gray, size) pair per zone;
// *max_region = the largest zone); rb_fill_glszm finishes it.
int segment_glszm(const void* lev, int level_bytes, const int* size, int nd, int Ng, int force2D, int force2Ddimension,
                  int* max_region, void** handle, cudaStream_t st) {
  SegmentGeometry sg;
  const int one[1] = {1};
  // the unidirectional distance-1 offsets: union-find joins each neighbour pair once
  const int rc = segment_geometry(size, nd, one, 1, false, force2D, force2Ddimension, Ng, NA_MAX, nullptr, sg);
  if (rc) return rc;
  std::unique_ptr<GlszmHandle> H(new GlszmHandle);   // handed to the caller only on success
  H->st = st;
  const long long n = sg.n;
  const Vol V{sg.Z, sg.Y, sg.X};
  const int grid = grid_for(n, 256, 8);
  DevBuf L, sz, scal;   // scal: [0] zones, [1] largest zone
  RB_CUDA(L.alloc(n * 4));
  RB_CUDA(sz.alloc(n * 4));
  RB_CUDA(scal.alloc(8));
  RB_CUDA(H->zones.alloc(sizeof(int) * 2 * (size_t)n));
  RB_CUDA(cudaMemsetAsync(sz.p, 0, n * 4, st));
  RB_CUDA(cudaMemsetAsync(scal.p, 0, 8, st));
  unsigned *d_sz = sz.as<unsigned>(), *sc = scal.as<unsigned>();
  int* zones = H->zones.as<int>();
  if (level_bytes == 1) {
    ccl_init_kernel<uint8_t><<<grid, 256, 0, st>>>((const uint8_t*)lev, n, L.as<int>());
    ccl_merge_kernel<uint8_t><<<grid, 256, 0, st>>>((const uint8_t*)lev, V, sg.A, L.as<int>());
    ccl_count_kernel<<<grid, 256, 0, st>>>(L.as<int>(), n, d_sz);
    ccl_zones_kernel<uint8_t><<<grid, 256, 0, st>>>((const uint8_t*)lev, L.as<int>(), d_sz, n, zones, sc, sc + 1);
  } else {
    ccl_init_kernel<uint16_t><<<grid, 256, 0, st>>>((const uint16_t*)lev, n, L.as<int>());
    ccl_merge_kernel<uint16_t><<<grid, 256, 0, st>>>((const uint16_t*)lev, V, sg.A, L.as<int>());
    ccl_count_kernel<<<grid, 256, 0, st>>>(L.as<int>(), n, d_sz);
    ccl_zones_kernel<uint16_t><<<grid, 256, 0, st>>>((const uint16_t*)lev, L.as<int>(), d_sz, n, zones, sc, sc + 1);
  }
  RB_LAUNCH_CHECK();
  unsigned host_sc[2] = {0, 0};
  RB_CUDA(cudaMemcpyAsync(host_sc, sc, 8, cudaMemcpyDeviceToHost, st));
  RB_CUDA(cudaStreamSynchronize(st));
  H->nzones = host_sc[0];
  *max_region = (int)host_sc[1];
  *handle = H.release();
  return RB_OK;
}

}  // namespace rb
