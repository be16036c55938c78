// Voxel-based first-order feature maps.  Two kernels:
//   firstorder_kernel<WCAP>  any window (r <= 3, clipped radii, 16-bit levels): one thread per centre voxel, grid-stride,
//                            gathers its window of raw intensities + discretised levels and evaluates
//                            firstorder_voxel<> (firstorder.cuh)
//   firstorder_tiles_kernel  kernelRadius 1 on every axis with 8-bit levels: the full/deferred tiles of full_window_tiles
//                            (voxel_tiles.cuh).  A centre whose 27 window voxels are all in the volume, in the kernel
//                            mask, non-zero in level and not NaN runs firstorder_full_body; every other centre is drained
//                            through the generic gather + firstorder_voxel<27>.  Both give the same bits.
//   firstorder_wide_kernel   windows of 344 to 3375 positions (kernelRadius 4 to 7): one block per centre, the window
//                            in shared memory, a stable rank sort by the block (insertion sort on one thread when the
//                            window holds a NaN), block_compact_levels' classes.  The same bits as firstorder_voxel.
#include "common.cuh"
#include "firstorder.cuh"
#include "host_common.hpp"
#include "pixel.cuh"
#include "voxel_tiles.cuh"
#include "wide_window.cuh"

namespace rb {

struct FoParams {
  int Z, Y, X;
  long long sz, sy;    // element strides of the (contiguous) image, mask and level volumes
  int rz, ry, rx, z0, z1, out_z0, dtype, level_bytes;
  double shift, voxel_volume, init_value;
};

// the generic window of centre (z, y, x): the intensities of the in-volume, in-mask voxels and every position's level
// (0 = not in the kernel), then firstorder_voxel<WCAP>
template <int WCAP>
__device__ __forceinline__ void firstorder_generic(const void* __restrict__ img, const uint8_t* __restrict__ mask,
                                                   const void* __restrict__ lev, const FoParams& P, int z, int y, int x,
                                                   double* f) {
  double xs[WCAP];
  uint16_t w[WCAP];
  int n = 0, wn = 0;
  for (int dz = -P.rz; dz <= P.rz; dz++)
    for (int dy = -P.ry; dy <= P.ry; dy++)
      for (int dx = -P.rx; dx <= P.rx; dx++, wn++) {
        const int zz = z + dz, yy = y + dy, xx = x + dx;
        w[wn] = 0;
        if (zz < 0 || zz >= P.Z || yy < 0 || yy >= P.Y || xx < 0 || xx >= P.X) continue;
        const long long j = (long long)zz * P.sz + (long long)yy * P.sy + xx;
        if (mask && !mask[j]) continue;
        xs[n++] = load_f64(img, P.dtype, j);
        w[wn] = P.level_bytes == 1 ? (uint16_t)((const uint8_t*)lev)[j] : ((const uint16_t*)lev)[j];
      }
  firstorder_voxel<WCAP>(xs, n, w, wn, P.shift, P.voxel_volume, f);
}

// whether chunk voxel v gets maps: centers[] if given, else the kernel mask (everything when NULL)
__device__ __forceinline__ bool firstorder_center(const uint8_t* __restrict__ mask, const uint8_t* __restrict__ centers,
                                                  const ChunkVoxel& v) {
  return centers ? centers[v.vi] != 0 : (mask ? mask[v.vi] != 0 : true);
}

template <int WCAP>
__global__ void __launch_bounds__(128)
firstorder_kernel(const void* __restrict__ img, const uint8_t* __restrict__ mask, const uint8_t* __restrict__ centers,
                  const void* __restrict__ lev, FoParams P, double* __restrict__ out, long long fstride) {
  const long long plane = (long long)P.Y * P.X;
  const long long total = (long long)(P.z1 - P.z0) * plane;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const ChunkVoxel v = chunk_voxel(P, plane, P.z0, P.out_z0, t);
    if (!firstorder_center(mask, centers, v)) {
#pragma unroll
      for (int k = 0; k < FIRSTORDER_NF; k++) out[k * fstride + v.oi] = P.init_value;
      continue;
    }
    double f[FIRSTORDER_NF];
    firstorder_generic<WCAP>(img, mask, lev, P, v.z, v.y, v.x, f);
#pragma unroll
    for (int k = 0; k < FIRSTORDER_NF; k++) out[k * fstride + v.oi] = f[k];
  }
}

// the 27 intensities of a window whose positions are all inside the volume, to xv in window order; whether all are in
// the kernel mask (or it is NULL) and none is NaN
template <typename T>
__device__ __forceinline__ bool firstorder_load27(const T* __restrict__ img, const uint8_t* __restrict__ mask,
                                                  const FoParams& P, long long vi, double* xv) {
  bool ok = true;
  int p = 0;
#pragma unroll
  for (int dz = -1; dz <= 1; dz++)
#pragma unroll
    for (int dy = -1; dy <= 1; dy++)
#pragma unroll
      for (int dx = -1; dx <= 1; dx++, p++) {
        const long long j = vi + (long long)dz * P.sz + (long long)dy * P.sy + dx;
        if (mask) ok &= mask[j] != 0;
        xv[p] = (double)img[j];
        ok &= xv[p] == xv[p];
      }
  return ok;
}

__device__ __forceinline__ bool firstorder_load27(const void* img, const uint8_t* mask, const FoParams& P, long long vi,
                                                  double* xv) {
  switch (P.dtype) {
    case RB_DT_INT16: return firstorder_load27((const int16_t*)img, mask, P, vi, xv);
    case RB_DT_INT32: return firstorder_load27((const int32_t*)img, mask, P, vi, xv);
    case RB_DT_FLOAT32: return firstorder_load27((const float*)img, mask, P, vi, xv);
    case RB_DT_FLOAT64: return firstorder_load27((const double*)img, mask, P, vi, xv);
    case RB_DT_UINT8: return firstorder_load27((const uint8_t*)img, mask, P, vi, xv);
    case RB_DT_UINT16: return firstorder_load27((const uint16_t*)img, mask, P, vi, xv);
    default: return firstorder_load27((const long long*)img, mask, P, vi, xv);
  }
}

// 128 threads, 4 blocks per SM (<= 128 registers); the sorted windows live in shared memory, [rank][thread]
constexpr int FO_NT = 128;
template <int NT>
__global__ void __launch_bounds__(NT, 4)
firstorder_tiles_kernel(const void* __restrict__ img, const uint8_t* __restrict__ mask,
                        const uint8_t* __restrict__ centers, const uint8_t* __restrict__ lev,
                        const __grid_constant__ FoParams P, double* __restrict__ out, long long fstride) {
  __shared__ double scr[27 * NT];
  __shared__ long long defer[2 * NT];                              // chunk indices of the centres left to the generic body
  __shared__ unsigned ndefer;
  const int tid = threadIdx.x;
  if (tid == 0) ndefer = 0;
  __syncthreads();
  const long long plane = (long long)P.Y * P.X;
  full_window_tiles<NT>((long long)(P.z1 - P.z0) * plane, defer, ndefer,
    [&](long long t, bool live, auto defer_it) {
      if (!live) return;
      const ChunkVoxel v = chunk_voxel(P, plane, P.z0, P.out_z0, t);
      if (!firstorder_center(mask, centers, v)) {
#pragma unroll
        for (int k = 0; k < FIRSTORDER_NF; k++) out[k * fstride + v.oi] = P.init_value;
        return;
      }
      int wl[27];
      double xv[27];
      if (load_window27(lev, P, v.z, v.y, v.x, v.vi, true, wl, 1) && firstorder_load27(img, mask, P, v.vi, xv)) {
        double f[FIRSTORDER_NF];
        firstorder_full_body(xv, wl, P.shift, P.voxel_volume, scr + tid, NT, f);
#pragma unroll
        for (int k = 0; k < FIRSTORDER_NF; k++) out[k * fstride + v.oi] = f[k];
      } else {
        defer_it();
      }
    },
    [&](auto entry, bool live) {
      if (!live) return;
      const ChunkVoxel v = chunk_voxel(P, plane, P.z0, P.out_z0, entry());
      double f[FIRSTORDER_NF];
      firstorder_generic<27>(img, mask, lev, P, v.z, v.y, v.x, f);
#pragma unroll
      for (int k = 0; k < FIRSTORDER_NF; k++) out[k * fstride + v.oi] = f[k];
    });
}

constexpr int FO_WIDE_NT = 128;
// shared memory of a wide window of wn positions: intensities by position and sorted, level scratch, levels, membership
static int fo_wide_smem(int wn) { return wn * (8 + 8 + 4 + 4 + 4 + 2 + 2 + 1); }

__global__ void __launch_bounds__(FO_WIDE_NT)
firstorder_wide_kernel(const void* __restrict__ img, const uint8_t* __restrict__ mask, const uint8_t* __restrict__ centers,
                       const void* __restrict__ lev, const __grid_constant__ FoParams P, double* __restrict__ out,
                       long long fstride) {
  extern __shared__ __align__(8) uint8_t smem[];
  const int wn = (2 * P.rz + 1) * (2 * P.ry + 1) * (2 * P.rx + 1), tid = threadIdx.x;
  double* xw = (double*)smem;            // intensity at each window position (members only)
  double* xs = xw + wn;                  // the members' intensities in ascending order
  int* fq = (int*)(xs + wn);
  int* val = fq + wn;
  int* cnt = val + wn;
  uint16_t* w = (uint16_t*)(cnt + wn);
  uint16_t* lidx = w + wn;
  uint8_t* in = (uint8_t*)(lidx + wn);   // in the volume and in the kernel mask
  __shared__ double s_f[FIRSTORDER_NF];
  __shared__ int s_n, s_nl, s_N, s_nan;
  const long long plane = (long long)P.Y * P.X;
  const long long total = (long long)(P.z1 - P.z0) * plane;
  for (long long t = blockIdx.x; t < total; t += gridDim.x) {         // block-uniform
    const ChunkVoxel v = chunk_voxel(P, plane, P.z0, P.out_z0, t);
    if (!firstorder_center(mask, centers, v)) {
      if (tid < FIRSTORDER_NF) out[tid * fstride + v.oi] = P.init_value;
      continue;
    }
    if (tid == 0) { s_n = 0; s_N = 0; s_nan = 0; }
    __syncthreads();
    int nloc = 0, Nloc = 0;
    bool nan = false;
    for (int p = tid; p < wn; p += FO_WIDE_NT) {        // firstorder_generic's gather, by position
      const WindowOffset o(p, P.rz, P.ry, P.rx);
      const int zz = v.z + o.dz, yy = v.y + o.dy, xx = v.x + o.dx;
      bool m = zz >= 0 && zz < P.Z && yy >= 0 && yy < P.Y && xx >= 0 && xx < P.X;
      const long long j = m ? (long long)zz * P.sz + (long long)yy * P.sy + xx : 0;
      if (m && mask && !mask[j]) m = false;
      in[p] = m;
      w[p] = 0;
      cnt[p] = 0;
      if (m) {
        xw[p] = load_f64(img, P.dtype, j);
        nan |= xw[p] != xw[p];
        w[p] = P.level_bytes == 1 ? (uint16_t)((const uint8_t*)lev)[j] : ((const uint16_t*)lev)[j];
        nloc++;
        Nloc += w[p] != 0;
      }
    }
    if (nloc) atomicAdd(&s_n, nloc);
    if (Nloc) atomicAdd(&s_N, Nloc);
    if (nan) s_nan = 1;
    __syncthreads();
    const int n = s_n;
    if (!s_nan) {
      // stable rank: #{members before j with x <= x_j} + #{members after j with x < x_j}, the insertion sort's position
      for (int jp = tid; jp < wn; jp += FO_WIDE_NT) {
        if (!in[jp]) continue;
        const double xj = xw[jp];
        int r = 0;
        for (int i = 0; i < jp; i++) r += in[i] && xw[i] <= xj;
        for (int i = jp + 1; i < wn; i++) r += in[i] && xw[i] < xj;
        xs[r] = xj;
      }
    } else if (tid == 0) {
      int k = 0;
      for (int p = 0; p < wn; p++) if (in[p]) xs[k++] = xw[p];
      fo_insertion_sort(xs, n);
    }
    const int nl = block_compact_levels(w, wn, val, lidx, fq, s_nl);
    for (int p = tid; p < wn; p += FO_WIDE_NT)
      if (lidx[p] != NOLEV) atomicAdd(&cnt[lidx[p]], 1);
    __syncthreads();
    if (tid == 0) {
      double ent, uni;
      fo_level_classes(cnt, nl, s_N, ent, uni);
      firstorder_sorted(xs, n, ent, uni, P.shift, P.voxel_volume, s_f);
    }
    __syncthreads();
    if (tid < FIRSTORDER_NF) out[tid * fstride + v.oi] = s_f[tid];
    __syncthreads();
  }
}

static FoParams fo_params(int dtype, int level_bytes, int Z, int Y, int X, int rz, int ry, int rx, double shift,
                          double voxel_volume, double init_value, int z0, int z1, int out_z0) {
  return FoParams{Z, Y, X, (long long)Y * X, X, rz, ry, rx, z0, z1, out_z0, dtype, level_bytes, shift, voxel_volume,
                  init_value};
}

int firstorder_fast_launch(const void* img, int dtype, const uint8_t* mask, const uint8_t* centers, const void* lev,
                           int Z, int Y, int X, double shift, double voxel_volume, double init_value, double* out,
                           long long fstride, int z0, int z1, int out_z0, cudaStream_t st) {
  const FoParams P = fo_params(dtype, 1, Z, Y, X, 1, 1, 1, shift, voxel_volume, init_value, z0, z1, out_z0);
  const long long total = (long long)(z1 - z0) * Y * X;
  if (total <= 0) return RB_OK;
  int grid = 0;
  RB_CUDA(resident_grid(firstorder_tiles_kernel<FO_NT>, FO_NT, 0, total, grid));
  firstorder_tiles_kernel<FO_NT><<<grid, FO_NT, 0, st>>>(img, mask, centers, (const uint8_t*)lev, P, out, fstride);
  RB_LAUNCH_CHECK();
  return RB_OK;
}

int firstorder_launch(const void* img, int dtype, const uint8_t* mask, const uint8_t* centers, const void* lev,
                      int level_bytes, int Z, int Y, int X, int rz, int ry, int rx, double shift, double voxel_volume,
                      double init_value, double* out, long long fstride, int z0, int z1, int out_z0, cudaStream_t st) {
  const FoParams P = fo_params(dtype, level_bytes, Z, Y, X, rz, ry, rx, shift, voxel_volume, init_value, z0, z1, out_z0);
  const long long total = (long long)(z1 - z0) * Y * X;
  if (total <= 0) return RB_OK;
  const int grid = grid_for(total, 128, 32);
  const int wcap = (2 * rz + 1) * (2 * ry + 1) * (2 * rx + 1);
  if (wcap <= 27) firstorder_kernel<27><<<grid, 128, 0, st>>>(img, mask, centers, lev, P, out, fstride);
  else if (wcap <= 125) firstorder_kernel<125><<<grid, 128, 0, st>>>(img, mask, centers, lev, P, out, fstride);
  else if (wcap <= 343) firstorder_kernel<343><<<grid, 128, 0, st>>>(img, mask, centers, lev, P, out, fstride);
  else return fail(RB_ERR_UNSUPPORTED, "kernelRadius > 3 is outside the implemented envelope");
  RB_LAUNCH_CHECK();
  return RB_OK;
}

int firstorder_wide_launch(const void* img, int dtype, const uint8_t* mask, const uint8_t* centers, const void* lev,
                           int level_bytes, int Z, int Y, int X, int rz, int ry, int rx, double shift, double voxel_volume,
                           double init_value, double* out, long long fstride, int z0, int z1, int out_z0, cudaStream_t st) {
  const FoParams P = fo_params(dtype, level_bytes, Z, Y, X, rz, ry, rx, shift, voxel_volume, init_value, z0, z1, out_z0);
  const long long total = (long long)(z1 - z0) * Y * X;
  if (total <= 0) return RB_OK;
  const int smem = fo_wide_smem((2 * rz + 1) * (2 * ry + 1) * (2 * rx + 1));
  RB_CUDA(set_max_dynamic_smem(firstorder_wide_kernel, fo_wide_smem(WIDE_WCAP_MAX)));
  int per_sm = 0;
  RB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, firstorder_wide_kernel, FO_WIDE_NT, smem));
  long long grid = (long long)sm_count() * (per_sm > 0 ? per_sm : 1);
  if (grid > total) grid = total;
  firstorder_wide_kernel<<<(int)grid, FO_WIDE_NT, smem, st>>>(img, mask, centers, lev, P, out, fstride);
  RB_LAUNCH_CHECK();
  return RB_OK;
}

}  // namespace rb
