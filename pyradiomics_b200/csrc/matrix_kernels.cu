// Texture-MATRIX builders (the cMatrices API surface): what reference radiomics/src/cmatrices.c
// computes, segment-based (one matrix for the whole ROI) and voxel-batched (one dense matrix per
// listed voxel, reference radiomics/src/_cmatrices.c:203-207 etc.).
//
//   segment mode : one thread per voxel, integer counts accumulated with atomics into a uint32
//                  histogram (privatised in shared memory when it fits), converted to the
//                  reference's float64 layout at the end; GLSZM = union-find connected-component
//                  labelling (26-neighbourhood, equal gray level) + zone-size histogram.
//   voxel batch  : one thread per listed voxel writes its private dense matrix (no atomics); this
//                  is the API-compatibility path -- the product's voxel-based features never
//                  materialise these (see voxel_kernels.cu / voxel_fast.cu).
#include "common.cuh"
#include "host_common.hpp"
#include "vox_features.cuh"

namespace rb {

struct AngleSet {
  int na;
  int8_t a[NA_MAX][3];
};

struct Vol {
  int Z, Y, X;
  __host__ __device__ long long n() const { return (long long)Z * Y * X; }
  __device__ bool in(int z, int y, int x) const { return z >= 0 && z < Z && y >= 0 && y < Y && x >= 0 && x < X; }
  __device__ long long idx(int z, int y, int x) const { return ((long long)z * Y + y) * X + x; }
};

static int grid_of(long long n, int block, int per_sm) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  long long need = (n + block - 1) / block, cap = (long long)sms * per_sm;
  return (int)(need < cap ? (need < 1 ? 1 : need) : cap);
}

// ------------------------------------------------------------------------------- segment mode
// GLCM / GLDM share the "histogram of (voxel, neighbour) events" shape.  hist is uint32, zeroed.
template <typename T, bool SHARED>
__global__ void __launch_bounds__(256)
seg_glcm_kernel(const T* __restrict__ lev, Vol V, const __grid_constant__ AngleSet A, int Ng, unsigned* __restrict__ hist) {
  extern __shared__ unsigned sh[];
  const int nbins = Ng * Ng * A.na;
  if (SHARED) { for (int i = threadIdx.x; i < nbins; i += blockDim.x) sh[i] = 0; __syncthreads(); }
  unsigned* h = SHARED ? sh : hist;
  const long long n = V.n(), plane = (long long)V.Y * V.X;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const int gi = lev[t];
    if (!gi) continue;
    const int z = (int)(t / plane), rem = (int)(t % plane), y = rem / V.X, x = rem % V.X;
    for (int a = 0; a < A.na; a++) {
      const int z2 = z + A.a[a][0], y2 = y + A.a[a][1], x2 = x + A.a[a][2];
      if (!V.in(z2, y2, x2)) continue;
      const int gj = lev[V.idx(z2, y2, x2)];
      if (gj) atomicAdd(&h[((gi - 1) * Ng + (gj - 1)) * A.na + a], 1u);
    }
  }
  if (SHARED) {
    __syncthreads();
    for (int i = threadIdx.x; i < nbins; i += blockDim.x) if (sh[i]) atomicAdd(&hist[i], sh[i]);
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
seg_gldm_kernel(const T* __restrict__ lev, Vol V, const __grid_constant__ AngleSet A, int Ng, int alpha,
                unsigned* __restrict__ hist) {
  const long long n = V.n(), plane = (long long)V.Y * V.X;
  const int ncol = 2 * A.na + 1;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const int gi = lev[t];
    if (!gi) continue;
    const int z = (int)(t / plane), rem = (int)(t % plane), y = rem / V.X, x = rem % V.X;
    int dep = 0;
    for (int a = 0; a < A.na; a++) {
      const int z2 = z + A.a[a][0], y2 = y + A.a[a][1], x2 = x + A.a[a][2];
      if (!V.in(z2, y2, x2)) continue;
      const int gj = lev[V.idx(z2, y2, x2)];
      if (!gj) continue;
      int d = gi - gj;
      if (d < 0) d = -d;
      if (d <= alpha) dep++;
    }
    atomicAdd(&hist[(gi - 1) * ncol + dep], 1u);
  }
}

// NGTDM: n_i exact; s_i = sum |g - sum/count| is accumulated as exact integers
// T[g][count] += |g*count - sum| and divided by count once at the end (deterministic).
template <typename T>
__global__ void __launch_bounds__(256)
seg_ngtdm_kernel(const T* __restrict__ lev, Vol V, const __grid_constant__ AngleSet A, int Ng,
                 unsigned long long* __restrict__ acc /* [Ng][na+2]: [0]=n_i, [1+c]=T_c */) {
  const long long n = V.n(), plane = (long long)V.Y * V.X;
  const int ncol = A.na + 2;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const int gi = lev[t];
    if (!gi) continue;
    const int z = (int)(t / plane), rem = (int)(t % plane), y = rem / V.X, x = rem % V.X;
    int cnt = 0; long long sum = 0;
    for (int a = 0; a < A.na; a++) {
      const int z2 = z + A.a[a][0], y2 = y + A.a[a][1], x2 = x + A.a[a][2];
      if (!V.in(z2, y2, x2)) continue;
      const int gj = lev[V.idx(z2, y2, x2)];
      if (gj) { cnt++; sum += gj; }
    }
    atomicAdd(&acc[(gi - 1) * ncol], 1ull);
    if (cnt) {
      long long num = (long long)gi * cnt - sum;
      if (num < 0) num = -num;
      if (num) atomicAdd(&acc[(gi - 1) * ncol + 1 + cnt], (unsigned long long)num);
    }
  }
}

__global__ void ngtdm_finish_kernel(const unsigned long long* __restrict__ acc, int Ng, int na, double* __restrict__ out) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= Ng) return;
  const int ncol = na + 2;
  double s = 0;
  for (int c = 1; c <= na; c++) s += (double)acc[g * ncol + 1 + c] / (double)c;
  out[g * 3 + 0] = (double)acc[g * ncol];
  out[g * 3 + 1] = s;
  out[g * 3 + 2] = (double)(g + 1);
}

// GLRLM: a thread owns (voxel, angle); it only works when the voxel starts a line for that angle.
template <typename T>
__global__ void __launch_bounds__(256)
seg_glrlm_kernel(const T* __restrict__ lev, Vol V, const __grid_constant__ AngleSet A, int Ng, int Nr,
                 unsigned* __restrict__ hist, unsigned* __restrict__ multi, int* __restrict__ status) {
  const long long n = V.n(), plane = (long long)V.Y * V.X;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const int z = (int)(t / plane), rem = (int)(t % plane), y = rem / V.X, x = rem % V.X;
    for (int a = 0; a < A.na; a++) {
      const int az = A.a[a][0], ay = A.a[a][1], ax = A.a[a][2];
      if (V.in(z - az, y - ay, x - ax)) continue;   // not the first voxel of its line
      int cz = z, cy = y, cx = x, gl = 0, rl = 0, elements = 0;
      while (V.in(cz, cy, cx)) {
        const int g = lev[V.idx(cz, cy, cx)];
        if (g) {
          elements++;
          if (!gl) { gl = g; rl = 0; }
          else if (g == gl) rl++;
          else {
            if (rl < Nr) atomicAdd(&hist[((gl - 1) * Nr + rl) * A.na + a], 1u); else atomicOr(status, 1);
            gl = g; rl = 0;
          }
        } else if (gl) {
          if (rl < Nr) atomicAdd(&hist[((gl - 1) * Nr + rl) * A.na + a], 1u); else atomicOr(status, 1);
          gl = 0; rl = 0;
        }
        cz += az; cy += ay; cx += ax;
      }
      if (gl) { if (rl < Nr) atomicAdd(&hist[((gl - 1) * Nr + rl) * A.na + a], 1u); else atomicOr(status, 1); }
      if (elements > 1) multi[a] = 1u;
    }
  }
}

// counts -> float64; optional GLRLM rule: angles without any multi-voxel line lose their
// run-length-1 column (cmatrices.c:524-534)
__global__ void counts_to_f64_kernel(const unsigned* __restrict__ hist, long long n, double* __restrict__ out,
                                     const unsigned* __restrict__ multi, int Nr, int na) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    double v = (double)hist[i];
    if (multi) {
      const int a = (int)(i % na), r = (int)((i / na) % Nr);
      if (r == 0 && !multi[a]) v = 0.0;
    }
    out[i] = v;
  }
}

// ---- GLSZM (segment): union-find connected components over equal-level 26/8-neighbours -----
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
__global__ void __launch_bounds__(256)
zones_fill_kernel(const int* __restrict__ zones, unsigned nzones, int Ng, int max_region, unsigned* __restrict__ hist,
                  int* __restrict__ status) {
  for (unsigned k = blockIdx.x * blockDim.x + threadIdx.x; k < nzones; k += gridDim.x * blockDim.x) {
    const int g = zones[2 * (size_t)k], s = zones[2 * (size_t)k + 1];
    if (g < 1 || g > Ng || s > max_region) { atomicOr(status, 1); continue; }
    atomicAdd(&hist[(size_t)(g - 1) * max_region + (s - 1)], 1u);
  }
}

// ------------------------------------------------------------------------------- voxel batches
struct BatchGeom {
  int Z, Y, X, rz, ry, rx, nvox;
};

template <typename T, int WCAP>
__device__ __forceinline__ void batch_window(const T* __restrict__ lev, const BatchGeom& G, const int* __restrict__ voxels,
                                             int v, uint16_t* w, VoxParams& P) {
  P.Z = G.Z; P.Y = G.Y; P.X = G.X; P.sy = G.X; P.sz = (long long)G.X * G.Y; P.rz = G.rz; P.ry = G.ry; P.rx = G.rx;
  load_window<T>(lev, P, voxels[v], voxels[G.nvox + v], voxels[2 * G.nvox + v], w);
}

// MODE 0 glcm, 1 gldm, 2 ngtdm, 3 glrlm
template <typename T, int WCAP, int MODE>
__global__ void __launch_bounds__(128)
batch_matrix_kernel(const T* __restrict__ lev, BatchGeom G, const int* __restrict__ voxels,
                    const __grid_constant__ AngleSet A, int Ng, int Nr, int alpha, double* __restrict__ out) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= G.nvox) return;
  uint16_t w[WCAP];
  VoxParams P;
  batch_window<T, WCAP>(lev, G, voxels, v, w, P);
  const WinGeom W(P);
  if (MODE == 0) {
    double* o = out + (size_t)v * Ng * Ng * A.na;
    for (int z = 0; z < W.wz; z++) for (int y = 0; y < W.wy; y++) for (int x = 0; x < W.wx; x++) {
      const int gi = w[W.idx(z, y, x)];
      if (!gi) continue;
      for (int a = 0; a < A.na; a++) {
        const int z2 = z + A.a[a][0], y2 = y + A.a[a][1], x2 = x + A.a[a][2];
        if (!W.inside(z2, y2, x2)) continue;
        const int gj = w[W.idx(z2, y2, x2)];
        if (gj) o[((size_t)(gi - 1) * Ng + (gj - 1)) * A.na + a] += 1.0;
      }
    }
  } else if (MODE == 1 || MODE == 2) {
    const int ncol = 2 * A.na + 1;
    double* o = out + (size_t)v * Ng * (MODE == 1 ? ncol : 3);
    if (MODE == 2) for (int g = 0; g < Ng; g++) o[g * 3 + 2] = g + 1;
    for (int z = 0; z < W.wz; z++) for (int y = 0; y < W.wy; y++) for (int x = 0; x < W.wx; x++) {
      const int gi = w[W.idx(z, y, x)];
      if (!gi) continue;
      int dep = 0; double cnt = 0, sum = 0;
      for (int a = 0; a < A.na; a++) {
        const int z2 = z + A.a[a][0], y2 = y + A.a[a][1], x2 = x + A.a[a][2];
        if (!W.inside(z2, y2, x2)) continue;
        const int gj = w[W.idx(z2, y2, x2)];
        if (!gj) continue;
        int d = gi - gj;
        if (d < 0) d = -d;
        if (d <= alpha) dep++;
        cnt += 1; sum += gj;
      }
      if (MODE == 1) o[(size_t)(gi - 1) * ncol + dep] += 1.0;
      else { o[(gi - 1) * 3] += 1.0; o[(gi - 1) * 3 + 1] += cnt == 0 ? 0.0 : fabs((double)gi - sum / cnt); }
    }
  } else {
    double* o = out + (size_t)v * Ng * Nr * A.na;
    for (int a = 0; a < A.na; a++) {
      const int az = A.a[a][0], ay = A.a[a][1], ax = A.a[a][2];
      bool multi = false;
      for (int z = 0; z < W.wz; z++) for (int y = 0; y < W.wy; y++) for (int x = 0; x < W.wx; x++) {
        if (W.inside(z - az, y - ay, x - ax)) continue;
        int cz = z, cy = y, cx = x, gl = 0, rl = 0, elements = 0;
        while (W.inside(cz, cy, cx)) {
          const int g = w[W.idx(cz, cy, cx)];
          if (g) {
            elements++;
            if (!gl) { gl = g; rl = 0; }
            else if (g == gl) rl++;
            else { o[((size_t)(gl - 1) * Nr + rl) * A.na + a] += 1.0; gl = g; rl = 0; }
          } else if (gl) { o[((size_t)(gl - 1) * Nr + rl) * A.na + a] += 1.0; gl = 0; rl = 0; }
          cz += az; cy += ay; cx += ax;
        }
        if (gl) o[((size_t)(gl - 1) * Nr + rl) * A.na + a] += 1.0;
        if (elements > 1) multi = true;
      }
      if (!multi) for (int g = 0; g < Ng; g++) o[((size_t)g * Nr) * A.na + a] = 0.0;
    }
  }
}

// GLSZM per listed voxel: zone list (gray,size) pairs, count per voxel, global max size
template <typename T, int WCAP>
__global__ void __launch_bounds__(128)
batch_glszm_zones_kernel(const T* __restrict__ lev, BatchGeom G, const int* __restrict__ voxels,
                         const __grid_constant__ AngleSet A, int* __restrict__ zones /*[nvox][2*WCAP]*/,
                         int* __restrict__ nz, unsigned* __restrict__ max_region) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= G.nvox) return;
  uint16_t w[WCAP], stack[WCAP];
  VoxParams P;
  batch_window<T, WCAP>(lev, G, voxels, v, w, P);
  const WinGeom W(P);
  int* zo = zones + (size_t)v * 2 * WCAP;
  int count = 0; unsigned mx = 0;
  for (int s = 0; s < W.n; s++) {
    const uint16_t gl = w[s];
    if (!gl) continue;
    int top = 0, region = 0;
    stack[top++] = (uint16_t)s; w[s] = 0;
    while (top) {
      const int k = stack[--top];
      region++;
      const int kz = k / (W.wy * W.wx), ky = (k / W.wx) % W.wy, kx = k % W.wx;
      for (int a = 0; a < A.na; a++) {
        const int z = kz + A.a[a][0], y = ky + A.a[a][1], x = kx + A.a[a][2];
        if (!W.inside(z, y, x)) continue;
        const int j = W.idx(z, y, x);
        if (w[j] == gl) { stack[top++] = (uint16_t)j; w[j] = 0; }
      }
    }
    zo[2 * count] = gl; zo[2 * count + 1] = region; count++;
    if ((unsigned)region > mx) mx = region;
  }
  nz[v] = count;
  atomicMax(max_region, mx);
}
__global__ void __launch_bounds__(128)
batch_glszm_fill_kernel(const int* __restrict__ zones, const int* __restrict__ nz, int nvox, int wcap, int Ng,
                        int max_region, double* __restrict__ out, int* __restrict__ status) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nvox) return;
  const int* zo = zones + (size_t)v * 2 * wcap;
  for (int k = 0; k < nz[v]; k++) {
    const int g = zo[2 * k], s = zo[2 * k + 1];
    if (g < 1 || g > Ng || s > max_region) { atomicOr(status, 1); continue; }
    out[((size_t)v * Ng + (g - 1)) * max_region + (s - 1)] += 1.0;
  }
}

// =============================================================================== host drivers
struct DevBuf {            // RAII for the host-buffer entry points
  void* p = nullptr;
  bool owned = true;       // false: a caller's device buffer (the *_dev entry points borrow the packed level volume)
  ~DevBuf() { if (p && owned) cudaFree(p); }
  int alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 1) == cudaSuccess ? 0 : -1; }
  template <typename U> U* as() { return (U*)p; }
};

int pack_levels(const int32_t* image, const uint8_t* mask, long long n, int Ng, void* lev, uint32_t* presence,
                int* status, cudaStream_t st);

struct Prepared {
  int nd, Z, Y, X, f2, lb;
  long long n;
  DevBuf lev, status, vox;
  AngleSet A;
  int na;
  std::vector<int> ang_nd;   // Na x nd, as the reference returns them
};

// common front end: shapes, angles, upload + pack (range check), optional voxel list upload
static int prepare(const int32_t* image, const uint8_t* mask, const int* size, int nd, const int* distances, int ndist,
                   bool bidirectional, int Ng, int force2D, int force2Ddimension, const int* voxels, int nvox,
                   int kernelRadius, Prepared& R, const void* levels_dev = nullptr) {
  if (!size || (nd != 2 && nd != 3)) return fail(RB_ERR_ARG, "image/mask must be 2-D or 3-D");
  if (Ng < 1 || Ng > 65535) return fail(RB_ERR_UNSUPPORTED, "Ng=%d outside 1..65535", Ng);
  if (voxels && kernelRadius <= 0) return fail(RB_ERR_ARG, "Expecting kernelRadius > 0");
  R.nd = nd;
  R.Z = nd == 3 ? size[0] : 1; R.Y = size[nd - 2]; R.X = size[nd - 1];
  R.n = (long long)R.Z * R.Y * R.X;
  if (R.n <= 0 || R.n >= (1ll << 31)) return fail(RB_ERR_UNSUPPORTED, "volume must have 1..2^31-1 voxels");
  const int f2_nd = force2D ? force2Ddimension : -1;
  R.f2 = f2_nd < 0 ? -1 : f2_nd + (3 - nd);
  R.na = generate_angles(size, nd, distances, ndist, bidirectional, f2_nd, R.ang_nd);
  if (R.na <= 0) return fail(RB_ERR_ARG, "Error getting angle count.");
  if (R.na > NA_MAX) return fail(RB_ERR_UNSUPPORTED, "more than %d angles", NA_MAX);
  R.A.na = R.na;
  for (int a = 0; a < R.na; a++)
    for (int d = 0; d < 3; d++) R.A.a[a][d] = d < 3 - nd ? 0 : (int8_t)R.ang_nd[a * nd + d - (3 - nd)];
  R.lb = Ng <= 255 ? 1 : 2;
  DevBuf dimg, dmsk;
  if (R.status.alloc(16)) return fail(RB_ERR_NOMEM, "device allocation failed");
  RB_CUDA(cudaMemsetAsync(R.status.p, 0, 16, 0));
  if (levels_dev) {                                  // device-resident packed levels (rb_pack_levels_dev), borrowed
    R.lev.p = const_cast<void*>(levels_dev);
    R.lev.owned = false;
  } else {
    if (!image || !mask) return fail(RB_ERR_ARG, "image/mask must be 2-D or 3-D");
    if (dimg.alloc(R.n * 4) || dmsk.alloc(R.n) || R.lev.alloc(R.n * R.lb)) return fail(RB_ERR_NOMEM, "device allocation failed");
    RB_CUDA(cudaMemcpyAsync(dimg.p, image, R.n * 4, cudaMemcpyHostToDevice, 0));
    RB_CUDA(cudaMemcpyAsync(dmsk.p, mask, R.n, cudaMemcpyHostToDevice, 0));
    int rc = pack_levels(dimg.as<int32_t>(), dmsk.as<uint8_t>(), R.n, Ng, R.lev.p, nullptr, R.status.as<int>(), 0);
    if (rc) return rc;
  }
  if (voxels) {
    if (nvox < 1) return fail(RB_ERR_ARG, "empty voxel list");
    std::vector<int> v3((size_t)3 * nvox, 0);
    for (int d = 0; d < nd; d++) memcpy(&v3[(size_t)(d + 3 - nd) * nvox], voxels + (size_t)d * nvox, sizeof(int) * nvox);
    for (int d = 0; d < nd; d++)
      for (int v = 0; v < nvox; v++) {
        int c = voxels[(size_t)d * nvox + v];
        if (c < 0 || c >= size[d]) return fail(RB_ERR_ARG, "voxel index out of range");
      }
    if (R.vox.alloc(sizeof(int) * 3 * (size_t)nvox)) return fail(RB_ERR_NOMEM, "device allocation failed");
    RB_CUDA(cudaMemcpyAsync(R.vox.p, v3.data(), sizeof(int) * 3 * (size_t)nvox, cudaMemcpyHostToDevice, 0));
    RB_CUDA(cudaStreamSynchronize(0));   // v3 is a temporary
  }
  RB_CUDA(cudaStreamSynchronize(0));     // dimg/dmsk go out of scope
  return RB_OK;
}

static int check_status(Prepared& R, const char* what) {
  int st[4] = {0, 0, 0, 0};
  RB_CUDA(cudaMemcpy(st, R.status.p, sizeof st, cudaMemcpyDeviceToHost));
  if (st[0] & 1) return fail(RB_ERR_LEVEL_RANGE, "Calculation of %s Failed: gray level outside 1..Ng inside the mask", what);
  if (st[1] & 1) return fail(RB_ERR_LEVEL_RANGE, "Calculation of %s Failed: index out of range", what);
  return RB_OK;
}

static BatchGeom batch_geom(const Prepared& R, int kernelRadius, int nvox) {
  BatchGeom G;
  G.Z = R.Z; G.Y = R.Y; G.X = R.X; G.nvox = nvox;
  G.rz = (R.f2 == 0 || R.nd == 2) ? 0 : kernelRadius;
  G.ry = R.f2 == 1 ? 0 : kernelRadius;
  G.rx = R.f2 == 2 ? 0 : kernelRadius;
  return G;
}

template <typename T, int MODE>
static int launch_batch(const Prepared& R, const BatchGeom& G, int Ng, int Nr, int alpha, double* out) {
  const int cap = (2 * G.rz + 1) * (2 * G.ry + 1) * (2 * G.rx + 1);
  const int grid = (G.nvox + 127) / 128;
  const T* lev = (const T*)R.lev.p;
  const int* vox = (const int*)R.vox.p;
  if (cap <= 27) batch_matrix_kernel<T, 27, MODE><<<grid, 128>>>(lev, G, vox, R.A, Ng, Nr, alpha, out);
  else if (cap <= 125) batch_matrix_kernel<T, 125, MODE><<<grid, 128>>>(lev, G, vox, R.A, Ng, Nr, alpha, out);
  else if (cap <= 343) batch_matrix_kernel<T, 343, MODE><<<grid, 128>>>(lev, G, vox, R.A, Ng, Nr, alpha, out);
  else return fail(RB_ERR_UNSUPPORTED, "kernelRadius > 3 is outside the implemented envelope");
  RB_LAUNCH_CHECK();
  return RB_OK;
}

// one driver for GLCM (mode 0) / GLDM (1) / NGTDM (2) / GLRLM (3)
int segment_tile_matrices(const uint8_t* lev, int nd, int Z, int Y, int X, const int* distances, int ndist, int Ng, int alpha,
                          int force2D, int force2Ddimension, double* glcm_host, double* gldm_host, double* ngtdm_host,
                          int* angles_out, int* na_out, cudaStream_t st);
int segment_glrlm(const void* lev, int level_bytes, int nd, int Z, int Y, int X, int Ng, int Nr, int force2D, int force2Ddimension,
                  double* glrlm_host, int* angles_out, int* na_out, cudaStream_t st);

static bool legacy_segment_kernels() {          // B200_SEG_LEGACY=1: round 1's kernels (cross-check in the tests)
  const char* e = getenv("B200_SEG_LEGACY");
  return e && e[0] == '1';
}

int calculate_matrix_host(int mode, const int32_t* image, const uint8_t* mask, const int* size, int nd,
                          const int* distances, int ndist, int Ng, int Nr, int alpha, int force2D, int force2Ddimension,
                          int kernelRadius, const int* voxels, int nvox, double* out_host, int* angles_out, int* na_out,
                          const void* levels_dev) {
  static const char* names[] = {"GLCM", "GLDM", "NGTDM", "GLRLM"};
  Prepared R;
  const int one[1] = {1};
  const bool bidir = mode == 1 || mode == 2;
  int rc = prepare(image, mask, size, nd, mode == 3 ? one : distances, mode == 3 ? 1 : ndist, bidir, Ng, force2D,
                   force2Ddimension, voxels, nvox, kernelRadius, R, levels_dev);
  if (rc) return rc;
  if (!voxels && !legacy_segment_kernels()) {
    // segment mode: the tile-staged fused kernel (8-bit levels, offsets up to 3) / the run-end GLRLM kernel
    int dmax = 0;
    for (int i = 0; i < ndist; i++) dmax = distances[i] > dmax ? distances[i] : dmax;
    if (mode == 3) {
      rc = segment_glrlm(R.lev.p, R.lb, nd, R.Z, R.Y, R.X, Ng, Nr, force2D, force2Ddimension, out_host, angles_out, na_out, 0);
      if (rc) return rc;
      return check_status(R, names[mode]);
    }
    if (R.lb == 1 && dmax <= 3) {
      rc = segment_tile_matrices(R.lev.as<uint8_t>(), nd, R.Z, R.Y, R.X, distances, ndist, Ng, alpha, force2D, force2Ddimension,
                                 mode == 0 ? out_host : nullptr, mode == 1 ? out_host : nullptr, mode == 2 ? out_host : nullptr,
                                 nullptr, nullptr, 0);
      if (rc == RB_OK) {
        if (na_out) *na_out = R.na;
        if (angles_out) memcpy(angles_out, R.ang_nd.data(), sizeof(int) * R.ang_nd.size());
        return check_status(R, names[mode]);
      }
      if (rc != RB_ERR_UNSUPPORTED) return rc;        // (too many levels for the shared-memory histograms: round 1's kernels)
    }
  }
  if (na_out) *na_out = R.na;
  if (angles_out) memcpy(angles_out, R.ang_nd.data(), sizeof(int) * R.ang_nd.size());
  const int nv = voxels ? nvox : 1;
  size_t per = mode == 0 ? (size_t)Ng * Ng * R.na : mode == 1 ? (size_t)Ng * (2 * R.na + 1) : mode == 2 ? (size_t)Ng * 3
                                                                                                  : (size_t)Ng * Nr * R.na;
  if (mode == 3 && Nr < 1) return fail(RB_ERR_ARG, "Nr must be >= 1");
  DevBuf dout;
  if (dout.alloc(sizeof(double) * per * nv)) return fail(RB_ERR_NOMEM, "device allocation of %zu matrix bytes failed", sizeof(double) * per * nv);
  RB_CUDA(cudaMemsetAsync(dout.p, 0, sizeof(double) * per * nv, 0));
  double* out = dout.as<double>();
  if (voxels) {
    BatchGeom G = batch_geom(R, kernelRadius, nvox);
#define RB_B(MODE) (R.lb == 1 ? launch_batch<uint8_t, MODE>(R, G, Ng, Nr, alpha, out) : launch_batch<uint16_t, MODE>(R, G, Ng, Nr, alpha, out))
    rc = mode == 0 ? RB_B(0) : mode == 1 ? RB_B(1) : mode == 2 ? RB_B(2) : RB_B(3);
#undef RB_B
    if (rc) return rc;
  } else {
    Vol V{R.Z, R.Y, R.X};
    const int grid = grid_of(R.n, 256, 8);
    DevBuf hist;
    int* status = R.status.as<int>();
    if (mode == 2) {
      const size_t nb = (size_t)Ng * (R.na + 2);
      if (hist.alloc(nb * 8)) return fail(RB_ERR_NOMEM, "device allocation failed");
      RB_CUDA(cudaMemsetAsync(hist.p, 0, nb * 8, 0));
      if (R.lb == 1) seg_ngtdm_kernel<uint8_t><<<grid, 256>>>(R.lev.as<uint8_t>(), V, R.A, Ng, hist.as<unsigned long long>());
      else seg_ngtdm_kernel<uint16_t><<<grid, 256>>>(R.lev.as<uint16_t>(), V, R.A, Ng, hist.as<unsigned long long>());
      RB_LAUNCH_CHECK();
      ngtdm_finish_kernel<<<(Ng + 127) / 128, 128>>>(hist.as<unsigned long long>(), Ng, R.na, out);
      RB_LAUNCH_CHECK();
    } else {
      DevBuf multi;
      if (hist.alloc(per * 4) || multi.alloc(4 * (size_t)R.na)) return fail(RB_ERR_NOMEM, "device allocation failed");
      RB_CUDA(cudaMemsetAsync(hist.p, 0, per * 4, 0));
      RB_CUDA(cudaMemsetAsync(multi.p, 0, 4 * (size_t)R.na, 0));
      unsigned* h = hist.as<unsigned>();
      if (mode == 0) {
        const size_t shbytes = per * 4;
        const bool sh = shbytes <= 160 * 1024;
        if (sh) {
          if (R.lb == 1) { cudaFuncSetAttribute(seg_glcm_kernel<uint8_t, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shbytes);
                           seg_glcm_kernel<uint8_t, true><<<grid_of(R.n, 256, 1), 256, shbytes>>>(R.lev.as<uint8_t>(), V, R.A, Ng, h); }
          else { cudaFuncSetAttribute(seg_glcm_kernel<uint16_t, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shbytes);
                 seg_glcm_kernel<uint16_t, true><<<grid_of(R.n, 256, 1), 256, shbytes>>>(R.lev.as<uint16_t>(), V, R.A, Ng, h); }
        } else {
          if (R.lb == 1) seg_glcm_kernel<uint8_t, false><<<grid, 256>>>(R.lev.as<uint8_t>(), V, R.A, Ng, h);
          else seg_glcm_kernel<uint16_t, false><<<grid, 256>>>(R.lev.as<uint16_t>(), V, R.A, Ng, h);
        }
      } else if (mode == 1) {
        if (R.lb == 1) seg_gldm_kernel<uint8_t><<<grid, 256>>>(R.lev.as<uint8_t>(), V, R.A, Ng, alpha, h);
        else seg_gldm_kernel<uint16_t><<<grid, 256>>>(R.lev.as<uint16_t>(), V, R.A, Ng, alpha, h);
      } else {
        if (R.lb == 1) seg_glrlm_kernel<uint8_t><<<grid, 256>>>(R.lev.as<uint8_t>(), V, R.A, Ng, Nr, h, multi.as<unsigned>(), status + 1);
        else seg_glrlm_kernel<uint16_t><<<grid, 256>>>(R.lev.as<uint16_t>(), V, R.A, Ng, Nr, h, multi.as<unsigned>(), status + 1);
      }
      RB_LAUNCH_CHECK();
      counts_to_f64_kernel<<<grid_of((long long)per, 256, 8), 256>>>(h, (long long)per, out, mode == 3 ? multi.as<unsigned>() : nullptr, Nr, R.na);
      RB_LAUNCH_CHECK();
      RB_CUDA(cudaStreamSynchronize(0));
    }
  }
  rc = check_status(R, names[mode]);
  if (rc) return rc;
  RB_CUDA(cudaMemcpy(out_host, out, sizeof(double) * per * nv, cudaMemcpyDeviceToHost));
  return RB_OK;
}

// ---- GLSZM two-phase --------------------------------------------------------------------
struct GlszmHandle {
  bool batch;
  int nvox, wcap, Ng;
  unsigned nzones;
  void* zones = nullptr;   // segment: int[2*nzones]; batch: int[nvox][2*wcap]
  void* nz = nullptr;      // batch: int[nvox]
  ~GlszmHandle() { cudaFree(zones); cudaFree(nz); }
};

int glszm_zones_host(const int32_t* image, const uint8_t* mask, const int* size, int nd, int Ng, int force2D,
                     int force2Ddimension, int kernelRadius, const int* voxels, int nvox, int* max_region_out,
                     void** handle_out, const void* levels_dev) {
  Prepared R;
  const int one[1] = {1};
  int rc = prepare(image, mask, size, nd, one, 1, true, Ng, force2D, force2Ddimension, voxels, nvox, kernelRadius, R, levels_dev);
  if (rc) return rc;
  rc = check_status(R, "GLSZM");
  if (rc) return rc;
  GlszmHandle* H = new GlszmHandle;
  H->Ng = Ng;
  DevBuf scal;   // [0] nzones, [1] max_region
  if (scal.alloc(8)) { delete H; return fail(RB_ERR_NOMEM, "device allocation failed"); }
  cudaMemsetAsync(scal.p, 0, 8, 0);
  unsigned* sc = scal.as<unsigned>();
  if (voxels) {
    BatchGeom G = batch_geom(R, kernelRadius, nvox);
    const int cap = (2 * G.rz + 1) * (2 * G.ry + 1) * (2 * G.rx + 1);
    const int wcap = cap <= 27 ? 27 : cap <= 125 ? 125 : 343;
    if (cap > 343) { delete H; return fail(RB_ERR_UNSUPPORTED, "kernelRadius > 3 is outside the implemented envelope"); }
    H->batch = true; H->nvox = nvox; H->wcap = wcap;
    if (cudaMalloc(&H->zones, sizeof(int) * 2 * (size_t)wcap * nvox) != cudaSuccess || cudaMalloc(&H->nz, sizeof(int) * (size_t)nvox) != cudaSuccess) {
      delete H; return fail(RB_ERR_NOMEM, "device allocation failed");
    }
    const int grid = (nvox + 127) / 128;
    const int* vox = (const int*)R.vox.p;
#define RB_Z(T, W) batch_glszm_zones_kernel<T, W><<<grid, 128>>>((const T*)R.lev.p, G, vox, R.A, (int*)H->zones, (int*)H->nz, sc + 1)
    if (R.lb == 1) { if (wcap == 27) RB_Z(uint8_t, 27); else if (wcap == 125) RB_Z(uint8_t, 125); else RB_Z(uint8_t, 343); }
    else { if (wcap == 27) RB_Z(uint16_t, 27); else if (wcap == 125) RB_Z(uint16_t, 125); else RB_Z(uint16_t, 343); }
#undef RB_Z
  } else {
    H->batch = false; H->nvox = 1; H->wcap = 0;
    Vol V{R.Z, R.Y, R.X};
    const int grid = grid_of(R.n, 256, 8);
    DevBuf L, sz;
    if (L.alloc(R.n * 4) || sz.alloc(R.n * 4)) { delete H; return fail(RB_ERR_NOMEM, "device allocation failed"); }
    cudaMemsetAsync(sz.p, 0, R.n * 4, 0);
    // the unidirectional half of the distance-1 neighbourhood = first half of the bidirectional set
    AngleSet half = R.A;
    half.na = R.A.na / 2;
    if (R.lb == 1) {
      ccl_init_kernel<uint8_t><<<grid, 256>>>(R.lev.as<uint8_t>(), R.n, L.as<int>());
      ccl_merge_kernel<uint8_t><<<grid, 256>>>(R.lev.as<uint8_t>(), V, half, L.as<int>());
    } else {
      ccl_init_kernel<uint16_t><<<grid, 256>>>(R.lev.as<uint16_t>(), R.n, L.as<int>());
      ccl_merge_kernel<uint16_t><<<grid, 256>>>(R.lev.as<uint16_t>(), V, half, L.as<int>());
    }
    ccl_count_kernel<<<grid, 256>>>(L.as<int>(), R.n, sz.as<unsigned>());
    // count roots first (cheap second pass) so the zone list is allocated exactly
    if (cudaMalloc(&H->zones, sizeof(int) * 2 * (size_t)R.n) != cudaSuccess) { delete H; return fail(RB_ERR_NOMEM, "device allocation failed"); }
    if (R.lb == 1) ccl_zones_kernel<uint8_t><<<grid, 256>>>(R.lev.as<uint8_t>(), L.as<int>(), sz.as<unsigned>(), R.n, (int*)H->zones, sc, sc + 1);
    else ccl_zones_kernel<uint16_t><<<grid, 256>>>(R.lev.as<uint16_t>(), L.as<int>(), sz.as<unsigned>(), R.n, (int*)H->zones, sc, sc + 1);
    cudaError_t e = cudaStreamSynchronize(0);
    if (e != cudaSuccess) { delete H; return fail(RB_ERR_CUDA, "GLSZM labelling: %s", cudaGetErrorString(e)); }
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { delete H; return fail(RB_ERR_CUDA, "GLSZM kernels: %s", cudaGetErrorString(e)); }
  unsigned host_sc[2] = {0, 0};
  e = cudaMemcpy(host_sc, sc, 8, cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) { delete H; return fail(RB_ERR_CUDA, "GLSZM: %s", cudaGetErrorString(e)); }
  H->nzones = host_sc[0];
  *max_region_out = (int)host_sc[1];
  *handle_out = H;
  return RB_OK;
}

int glszm_fill_host(void* handle, int Ng, int max_region, double* out_host) {
  GlszmHandle* H = (GlszmHandle*)handle;
  if (!H) return fail(RB_ERR_ARG, "null GLSZM handle");
  if (max_region < 1) max_region = 1;
  const size_t per = (size_t)Ng * max_region, tot = per * H->nvox;
  DevBuf dout, status;
  int rc = RB_OK;
  if (dout.alloc(tot * 8) || status.alloc(4)) { delete H; return fail(RB_ERR_NOMEM, "device allocation failed"); }
  cudaMemsetAsync(dout.p, 0, tot * 8, 0);
  cudaMemsetAsync(status.p, 0, 4, 0);
  if (H->batch) {
    batch_glszm_fill_kernel<<<(H->nvox + 127) / 128, 128>>>((const int*)H->zones, (const int*)H->nz, H->nvox, H->wcap, Ng, max_region, dout.as<double>(), status.as<int>());
  } else {
    DevBuf hist;
    if (hist.alloc(per * 4)) { delete H; return fail(RB_ERR_NOMEM, "device allocation failed"); }
    cudaMemsetAsync(hist.p, 0, per * 4, 0);
    if (H->nzones) zones_fill_kernel<<<grid_of(H->nzones, 256, 8), 256>>>((const int*)H->zones, H->nzones, Ng, max_region, hist.as<unsigned>(), status.as<int>());
    counts_to_f64_kernel<<<grid_of((long long)per, 256, 8), 256>>>(hist.as<unsigned>(), (long long)per, dout.as<double>(), nullptr, 1, 1);
    cudaStreamSynchronize(0);
  }
  int st = 0;
  cudaError_t e = cudaMemcpy(&st, status.p, 4, cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) rc = fail(RB_ERR_CUDA, "GLSZM fill: %s", cudaGetErrorString(e));
  else if (st) rc = fail(RB_ERR_LEVEL_RANGE, "Error filling GLSZM.");
  else if (cudaMemcpy(out_host, dout.p, tot * 8, cudaMemcpyDeviceToHost) != cudaSuccess) rc = fail(RB_ERR_CUDA, "GLSZM copy back failed");
  delete H;
  return rc;
}

void glszm_release(void* handle) { delete (GlszmHandle*)handle; }

}  // namespace rb
